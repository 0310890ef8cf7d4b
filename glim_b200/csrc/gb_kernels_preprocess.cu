// gb_kernels_preprocess.cu -- per-frame preprocess on the GPU (sm_90a): k-NN, covariance / normal
// estimation, voxel-grid downsampling.
//
// Replaces, at GLIM's call sites:
//   CloudPreprocessor::find_neighbors            src/glim/preprocess/cloud_preprocessor.cpp:190-221  (gtsam_points::KdTree::knn_search)
//   CloudCovarianceEstimation::estimate (PLANE)  src/glim/common/cloud_covariance_estimation.cpp:43-122, :181-196
//   gtsam_points::voxelgrid_sampling             src/glim/preprocess/cloud_preprocessor.cpp:108
// Oracles: go_knn_bruteforce, go_covariance_estimate, go_voxelgrid_sampling (oracle/glim_oracle.c).
// All three work in fp64 like the reference's host code (Vector4d / Matrix4d).
// The voxel grouping (sort, head flags, scan, voxel starts), the hash thinning and the device cloud build are shared with the
// voxel-map paths (gb_group_by_key, gb_group_starts, gb_thin, gb_cloud_build in gb_kernels_voxelmap.cu); the fp64 key kernel
// and the group means are this file's.
// The entry points gb_covariances, gb_find_neighbors, gb_cloud_estimate_covariances, gb_voxelgrid_sampling, gb_preprocess and
// gb_merge_frames are defined here.
#include "gb_internal.cuh"
#include "gb_cov_math.cuh"  // plane_covariance (shared with the host-compiled CPU test of the covariance arithmetic)

#include <cub/cub.cuh>
#include <cmath>
#include <string.h>
#include <algorithm>
#include <new>
#include <type_traits>

namespace {

// fp64 4x4 column-major covariance of the host layout
__device__ __forceinline__ void store_cov4x4(double* __restrict__ Co, const double (&C)[9]) {
  for (int e = 0; e < 16; e++) Co[e] = 0.0;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) Co[c * 4 + r] = C[r * 3 + c];
}

// ---------------------------------------------------------------------------------------------
// voxel-grid downsampling (fp64 coordinates, SURVEY C.2)
// ---------------------------------------------------------------------------------------------
__global__ void k_grid_keys(int n, const double4* __restrict__ pts, double inv_res, const int* __restrict__ keep, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double4 p = pts[i];
  unsigned long long key = kInvalidKey;
  if ((!keep || keep[i]) && isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    const double fx = floor(p.x * inv_res), fy = floor(p.y * inv_res), fz = floor(p.z * inv_res);
    if (fabs(fx) < 2e9 && fabs(fy) < 2e9 && fabs(fz) < 2e9) {
      unsigned long long k;
      if (gb_pack_key((int)fx, (int)fy, (int)fz, &k)) key = k;
    }
  }
  keys[i] = key;
  idx[i] = i;
}
// The fp64 mean of each voxel's members in sorted-slot order, for the voxel-grid downsampling and the frame merge: points,
// and the times, intensities and 6-entry covariances when given.  num_voxels = device count of voxels (the last element of
// the inclusive scan of gb_group_by_key).
__global__ void k_grid_means_counted(const int* __restrict__ num_voxels, const int* __restrict__ starts, const int* __restrict__ idx, const double4* __restrict__ pts, const double* __restrict__ times, const double* __restrict__ intens,
                                     const double* __restrict__ cov6, double4* __restrict__ out_pts, double* __restrict__ out_times, double* __restrict__ out_intens, double* __restrict__ out_cov6) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= *num_voxels) return;
  const int b = starts[v], e = starts[v + 1];
  double sx = 0, sy = 0, sz = 0, sw = 0, st = 0, si = 0, c[6] = {0, 0, 0, 0, 0, 0};
  for (int s = b; s < e; s++) {  // same sums in the same order as the oracle
    const int i = idx[s];
    const double4 p = pts[i];
    sx += p.x; sy += p.y; sz += p.z; sw += p.w;
    if (times) st += times[i];
    if (intens) si += intens[i];
    if (cov6)
      for (int m = 0; m < 6; m++) c[m] += cov6[6 * (size_t)i + m];
  }
  const int cnt = e - b;
  out_pts[v] = make_double4(sx / cnt, sy / cnt, sz / cnt, sw / cnt);
  if (times) out_times[v] = st / cnt;
  if (intens) out_intens[v] = si / cnt;
  if (cov6)
    for (int m = 0; m < 6; m++) out_cov6[6 * (size_t)v + m] = c[m] / cnt;
}

}  // namespace

gb_status gb_grid_keys(gb_ctx* ctx, int n, const double4* pts, double inv_res, const int* keep, unsigned long long* keys, int* idx) {
  return gb_launch(ctx, "k_grid_keys", k_grid_keys, (n + 255) / 256, 256, 0, n, pts, inv_res, keep, keys, idx);
}

// Returns launch(std::integral_constant<int, K>()) for the instantiated neighbour counts K of k_knn_pyramid.
template <typename Launch> static gb_status knn_dispatch(int k, Launch&& launch) {
  switch (k) {
#define KNN_CASE(K) case K: return launch(std::integral_constant<int, K>());
    KNN_CASE(1) KNN_CASE(2) KNN_CASE(3) KNN_CASE(4) KNN_CASE(5) KNN_CASE(6) KNN_CASE(7) KNN_CASE(8)
    KNN_CASE(9) KNN_CASE(10) KNN_CASE(12) KNN_CASE(15) KNN_CASE(16) KNN_CASE(20) KNN_CASE(24) KNN_CASE(32)
#undef KNN_CASE
  }
  gb_set_error("k = %d is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)", k);
  return GB_ERR_INVALID_ARGUMENT;
}
bool gb_knn_instantiated(int k) {
  return knn_dispatch(k, [](auto) { return GB_OK; }) == GB_OK;
}

size_t gb_cub_temp_bytes(size_t n_) {
  const int n = (int)n_;
  size_t sort_pairs = 0, sort_keys = 0, scan = 0, sum = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_pairs, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64);
  cub::DeviceRadixSort::SortKeys(nullptr, sort_keys, (unsigned long long*)nullptr, (unsigned long long*)nullptr, n, 0, 64);
  cub::DeviceScan::InclusiveSum(nullptr, scan, (int*)nullptr, (int*)nullptr, n);
  cub::DeviceReduce::Sum(nullptr, sum, (double*)nullptr, (double*)nullptr, n);
  return std::max({sort_pairs, sort_keys, scan, sum});
}

extern "C" gb_status gb_covariances(gb_ctx* ctx, size_t n, const double* xyzw, const int32_t* neighbors, int k_correspondences, int k_neighbors, double* normals4, double* cov4x4) {
  GB_REQUIRE(ctx, "null ctx");
  if (n == 0) return GB_OK;  // cloud_covariance_estimation.cpp:49-51
  GB_REQUIRE(xyzw && neighbors && normals4 && cov4x4, "null argument");
  GB_REQUIRE(k_neighbors > 0 && k_neighbors <= k_correspondences, "k_neighbors must be in [1, k_correspondences]");
  GB_REQUIRE(n < (size_t)1 << 30, "too many points");
  // the kernel gathers the points of the first k_neighbors entries of every row: an index outside [0, n) would be an
  // out-of-bounds device read
  for (size_t i = 0; i < n; i++)
    for (int j = 0; j < k_neighbors; j++) {
      const int32_t q = neighbors[i * (size_t)k_correspondences + j];
      GB_REQUIRE(q >= 0 && (size_t)q < n, "neighbour index out of range [0, n)");
    }
  GB_ENTER(ctx);
  double4 *d_pts, *d_nrm;
  int *d_nb, *d_cnt;
  double* d_cov;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_pts = cv.take<double4>(n);
    d_nb = cv.take<int>(n * k_correspondences);
    d_nrm = cv.take<double4>(n);
    d_cov = cv.take<double>(16 * n);
    d_cnt = cv.take<int>(1);
  }));
  const int count = (int)n;
  GB_CHECK(gb_upload(ctx, {{d_cnt, &count, sizeof(int)}, {d_pts, xyzw, sizeof(double4) * n}, {d_nb, neighbors, sizeof(int) * n * k_correspondences}}));
  GB_CHECK(gb_covariance_cloud(ctx, count, d_cnt, d_pts, d_nb, k_correspondences, k_neighbors, d_nrm, d_cov, gb_planes{}, gb_sort_tmp{}, nullptr));
  return gb_download(ctx, {{normals4, d_nrm, sizeof(double4) * n}, {cov4x4, d_cov, sizeof(double) * 16 * n}});
}

extern "C" gb_status gb_voxelgrid_sampling(gb_ctx* ctx, size_t n, const double* xyzw, const double* times, const double* intensities, double resolution, double* out_xyzw, double* out_times, double* out_intensities, size_t* num_out) {
  GB_REQUIRE(ctx && num_out, "null argument");
  *num_out = 0;
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw && out_xyzw && resolution > 0.0, "null argument");
  GB_ENTER(ctx);
  const size_t cub_b = gb_cub_temp_bytes(n);
  gb_sort_tmp t;
  double4 *d_pts, *d_opts;
  double *d_t, *d_i, *d_ot, *d_oi;
  int *d_flags, *d_pos, *d_starts;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    t = gb_take_sort_tmp(cv, n, cv.take<char>(cub_b), cub_b);
    d_pts = cv.take<double4>(n);
    d_opts = cv.take<double4>(n);
    d_t = cv.take<double>(n);
    d_i = cv.take<double>(n);
    d_ot = cv.take<double>(n);
    d_oi = cv.take<double>(n);
    d_flags = cv.take<int>(n + 1);
    d_pos = cv.take<int>(n + 1);
    d_starts = cv.take<int>(n + 1);
  }));
  GB_CHECK(gb_upload(ctx, {{d_pts, xyzw, sizeof(double4) * n}, {d_t, times, sizeof(double) * n}, {d_i, intensities, sizeof(double) * n}}));
  GB_CHECK(gb_grid_keys(ctx, (int)n, d_pts, 1.0 / resolution, nullptr, t.keys, t.idx));
  GB_CHECK(gb_group_by_key(ctx, (int)n, t, d_flags, d_pos));
  int V = 0;
  GB_CHECK(gb_download(ctx, {{&V, d_pos + (n - 1), sizeof(int)}}));
  if (V > 0) {
    GB_CHECK(gb_group_starts(ctx, (int)n, t, d_flags, d_pos, d_starts));
    GB_CHECK(gb_launch(ctx, "k_grid_means_counted", k_grid_means_counted, (n + 127) / 128, 128, 0, d_pos + (n - 1), d_starts, t.idx_s, d_pts, times ? d_t : nullptr,
                       intensities ? d_i : nullptr, nullptr, d_opts, d_ot, d_oi, nullptr));
    const size_t v = (size_t)V;
    GB_CHECK(gb_download(ctx, {{out_xyzw, d_opts, sizeof(double4) * v}, {times ? out_times : nullptr, d_ot, sizeof(double) * v},
                               {intensities ? out_intensities : nullptr, d_oi, sizeof(double) * v}}));
  }
  *num_out = (size_t)V;
  return GB_OK;
}

// =============================================================================================
// gb_preprocess: the whole per-frame preprocess on the device, without host round trips
//   CloudPreprocessor::preprocess_impl (src/glim/preprocess/cloud_preprocessor.cpp:92-188): downsample (voxel grid :108 or
//   random grid :104-106) -> finite + range gate (:116-128) -> crop box (:143-162) -> time order (:135-136) ->
//   global shutter (:138-140) -> k-NN (:182-183, :190-221)
//   + CloudCovarianceEstimation::estimate (src/glim/common/cloud_covariance_estimation.cpp:43-122; called on the preprocessed
//   frame at src/glim/odometry/odometry_estimation_imu.cpp:322-328) + PointCloudGPU::clone (odometry_estimation_gpu.cpp:96):
//   the fp32 planes of the gb_cloud are written straight from the covariance kernel's registers.
// One H2D of the raw scan, no host synchronisation until the point count is needed to size the cloud, optional D2H of
// the host-side products (PreprocessedFrame fields, covariances, normals).
// =============================================================================================
namespace {

// ---- Morton keys: one sort serves a whole pyramid of grids (cell size h0 * 4^level: a coarser cell is key >> 6 level) ----
__device__ __forceinline__ unsigned long long morton3(unsigned x, unsigned y, unsigned z) { return (gb_spread21(x) << 2) | (gb_spread21(y) << 1) | gb_spread21(z); }

constexpr int kMlLevels = 4;
constexpr double kMlOffset = 1048576.0;  // 2^20: coordinates are offset to [0, 2^21)
struct MlCell { unsigned long long key; int start; int pad; };
constexpr unsigned long long kMlEmpty = ~0ull;

__device__ __forceinline__ unsigned ml_hash(unsigned long long key, unsigned mask) { return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 32) & mask; }

// valid = device count of leading valid points (points [0, *valid) are considered; the rest get the invalid key)
__global__ void k_ml_keys(int n, const int* __restrict__ valid, const double4* __restrict__ pts, double inv_h0, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long key = kMlEmpty;
  if (i < *valid) {
    const double4 p = pts[i];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const double fx = floor(p.x * inv_h0) + kMlOffset, fy = floor(p.y * inv_h0) + kMlOffset, fz = floor(p.z * inv_h0) + kMlOffset;
      if (fx >= 0.0 && fx < 2097152.0 && fy >= 0.0 && fy < 2097152.0 && fz >= 0.0 && fz < 2097152.0) key = morton3((unsigned)fx, (unsigned)fy, (unsigned)fz);
    }
  }
  keys[i] = key;
  idx[i] = i;
}
__global__ void k_ml_gather(int n, const unsigned long long* __restrict__ keys_s, const int* __restrict__ idx_s, const double4* __restrict__ pts, double4* __restrict__ pts_s) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n && keys_s[s] != kMlEmpty) pts_s[s] = pts[idx_s[s]];
}
// every first point of a cell (at every level) registers the cell's start in that level's hash table
__global__ void k_ml_cells(int n, const unsigned long long* __restrict__ keys_s, MlCell* __restrict__ tables, unsigned table_size) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const unsigned long long key = keys_s[s];
  if (key == kMlEmpty) return;
  const unsigned long long prev = s > 0 ? keys_s[s - 1] : kMlEmpty;
#pragma unroll
  for (int l = 0; l < kMlLevels; l++) {
    const unsigned long long kl = key >> (6 * l);
    if (s > 0 && (prev >> (6 * l)) == kl) continue;
    MlCell* tab = tables + (size_t)l * table_size;
    unsigned slot = ml_hash(kl, table_size - 1);
    while (true) {
      const unsigned long long old = atomicCAS(&tab[slot].key, kMlEmpty, kl);
      if (old == kMlEmpty) { tab[slot].start = s; break; }
      slot = (slot + 1) & (table_size - 1);
    }
  }
}

template <int K>
__device__ __forceinline__ void knn_insert(double (&bd)[K], int (&bi)[K], int& cnt, double d, int j) {
  if (d < bd[K - 1] || (d == bd[K - 1] && j < bi[K - 1])) {
    double cd = d;
    int ci = j;
#pragma unroll
    for (int k = 0; k < K; k++) {
      if (cd < bd[k] || (cd == bd[k] && ci < bi[k])) {
        const double td = bd[k]; const int ti = bi[k];
        bd[k] = cd; bi[k] = ci; cd = td; ci = ti;
      }
    }
    cnt++;
  }
}

// Exact k-NN on the pyramid: a query searches the 3x3x3 block of cells around it at the finest level; every unseen point is
// then at least (1 + min(u, 1 - u)) * h away (u = position inside its cell), so the answer is complete as soon as the k-th
// best distance is within that bound.  Otherwise the query moves one level up (4x larger cells); after the coarsest level it
// scans all points.  Same un-contracted fp64 distance and (distance, index) tie rule as the oracle.
template <int K>
__global__ void __launch_bounds__(128) k_knn_pyramid(int n, const double4* __restrict__ pts_s, const unsigned long long* __restrict__ keys_s, const int* __restrict__ idx_s,
                                                     const MlCell* __restrict__ tables, unsigned table_size, double inv_h0, double h0, int* __restrict__ neighbors) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned long long key = keys_s[t];
  if (key == kMlEmpty) return;  // not a point of the frame (or a non-finite one: the caller pre-filled its row with itself)
  const int self = idx_s[t];
  const double4 p = pts_s[t];
  double bd[K];
  int bi[K];
  int cnt = 0;
  bool complete = false;
  const double px = p.x * inv_h0 + kMlOffset, py = p.y * inv_h0 + kMlOffset, pz = p.z * inv_h0 + kMlOffset;
  double scale = 1.0, h = h0;
  for (int l = 0; l < kMlLevels && !complete; l++, scale *= 0.25, h *= 4.0) {
#pragma unroll
    for (int k = 0; k < K; k++) { bd[k] = 1e300; bi[k] = 0x7fffffff; }
    cnt = 0;
    const double qx = px * scale, qy = py * scale, qz = pz * scale;
    const double fx = floor(qx), fy = floor(qy), fz = floor(qz);
    const int cx = (int)fx, cy = (int)fy, cz = (int)fz;
    const int cmax = (1 << (21 - 2 * l)) - 1;
    const MlCell* tab = tables + (size_t)l * table_size;
    for (int dx = -1; dx <= 1; dx++) {
      const int x = cx + dx;
      if (x < 0 || x > cmax) continue;
      for (int dy = -1; dy <= 1; dy++) {
        const int y = cy + dy;
        if (y < 0 || y > cmax) continue;
        for (int dz = -1; dz <= 1; dz++) {
          const int z = cz + dz;
          if (z < 0 || z > cmax) continue;
          const unsigned long long kl = morton3((unsigned)x, (unsigned)y, (unsigned)z);
          unsigned slot = ml_hash(kl, table_size - 1);
          int start = -1;
          while (true) {
            const unsigned long long tk = tab[slot].key;
            if (tk == kl) { start = tab[slot].start; break; }
            if (tk == kMlEmpty) break;
            slot = (slot + 1) & (table_size - 1);
          }
          if (start < 0) continue;
          for (int s = start; s < n; s++) {
            const unsigned long long ks = __ldg(&keys_s[s]);
            if (ks == kMlEmpty || (ks >> (6 * l)) != kl) break;
            const double4 q = pts_s[s];
            const double ex = p.x - q.x, ey = p.y - q.y, ez = p.z - q.z;
            const double d = __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
            knn_insert<K>(bd, bi, cnt, d, __ldg(&idx_s[s]));
          }
        }
      }
    }
    if (cnt >= K) {
      const double ux = qx - fx, uy = qy - fy, uz = qz - fz;
      const double m = 1.0 + fmin(fmin(fmin(ux, 1.0 - ux), fmin(uy, 1.0 - uy)), fmin(uz, 1.0 - uz));
      const double bound = m * h * (1.0 - 1e-12);
      if (bd[K - 1] <= bound * bound) complete = true;
    }
  }
  if (!complete) {  // isolated point: exact scan of all points
#pragma unroll
    for (int k = 0; k < K; k++) { bd[k] = 1e300; bi[k] = 0x7fffffff; }
    cnt = 0;
    for (int s = 0; s < n; s++) {
      if (__ldg(&keys_s[s]) == kMlEmpty) break;  // invalid keys sort last
      const double4 q = pts_s[s];
      const double ex = p.x - q.x, ey = p.y - q.y, ez = p.z - q.z;
      const double d = __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
      knn_insert<K>(bd, bi, cnt, d, __ldg(&idx_s[s]));
    }
  }
  const int found = min(cnt, K);
#pragma unroll
  for (int k = 0; k < K; k++) neighbors[(size_t)self * K + k] = k < found ? bi[k] : self;
}
__global__ void k_fill_self(int n, int k, int* __restrict__ neighbors) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < (size_t)n * k) neighbors[e] = (int)(e / k);
}

// ---- downsampling, filtering, time order ----
// random grid (gtsam_points::randomgrid_sampling, cloud_preprocessor.cpp:104-106): every voxel keeps at most
// ppv = ceil(rate * N / V) of its points.  Which ones is a draw from std::mt19937 in the reference (not reproducible, SURVEY
// C.2); here it is the ppv points with the smallest rg_hash(seed, index) (gb_vgicp_math.cuh) -- a fixed pseudo-random choice the
// oracle shares.
__global__ void k_randomgrid_select(int n, const int* __restrict__ num_voxels, const int* __restrict__ starts, const int* __restrict__ idx_s, double rate, unsigned long long seed, int* __restrict__ keep) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const int V = *num_voxels;
  if (v >= V) return;
  const int ppv = max(1, (int)ceil(rate * (double)n / (double)V));
  const int b = starts[v], e = starts[v + 1];
  if (e - b <= ppv) {
    for (int s = b; s < e; s++) keep[idx_s[s]] = 1;
    return;
  }
  // the ppv smallest hashes: threshold selection by repeated minimum (ppv is small: 1-4 at GLIM's settings)
  unsigned long long last = 0;
  int last_idx = -1;
  for (int r = 0; r < ppv; r++) {
    unsigned long long best = ~0ull;
    int best_i = -1;
    for (int s = b; s < e; s++) {
      const int i = idx_s[s];
      const unsigned long long hsh = rg_hash(seed, (unsigned)i);
      const bool after = (r == 0) || hsh > last || (hsh == last && i > last_idx);
      if (after && (hsh < best || (hsh == best && i < best_i))) { best = hsh; best_i = i; }
    }
    if (best_i < 0) break;
    keep[best_i] = 1;
    last = best; last_idx = best_i;
  }
}


struct FrameFilter {
  double near2, far2;
  int crop;  // 0 none, 1 box given in the lidar frame, 2 box given in the IMU frame (p_imu = T * p_lidar)
  double bmin[3], bmax[3];
  double T[12];  // rows of T_imu_lidar (3x4)
  int global_shutter;
};
// key = order-preserving bits of the time for the points that pass the gates, ~0 otherwise (sorted to the end, stable)
__global__ void k_filter_time_keys(int n_upper, const int* __restrict__ count_in, const int* __restrict__ keep, const double4* __restrict__ pts, const double* __restrict__ times, FrameFilter f,
                                   unsigned long long* __restrict__ keys, int* __restrict__ idx, int* __restrict__ count_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int ok = 0;
  if (i < n_upper) {
    unsigned long long key = ~0ull;
    if (i < *count_in && (!keep || keep[i])) {
      const double4 p = pts[i];
      const bool finite = isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && isfinite(p.w);          // :123 allFinite
      const double sq = __dadd_rn(__dadd_rn(__dmul_rn(p.x, p.x), __dmul_rn(p.y, p.y)), __dmul_rn(p.z, p.z));  // :124
      bool pass = finite && sq > f.near2 && sq < f.far2;                                             // :125
      if (pass && f.crop) {                                                                            // :143-162
        double x = p.x, y = p.y, z = p.z;
        if (f.crop == 2) {
          x = f.T[0] * p.x + f.T[1] * p.y + f.T[2] * p.z + f.T[3];
          y = f.T[4] * p.x + f.T[5] * p.y + f.T[6] * p.z + f.T[7];
          z = f.T[8] * p.x + f.T[9] * p.y + f.T[10] * p.z + f.T[11];
        }
        const bool inside = x >= f.bmin[0] && x <= f.bmax[0] && y >= f.bmin[1] && y <= f.bmax[1] && z >= f.bmin[2] && z <= f.bmax[2];
        pass = !inside;
      }
      if (pass) {
        const double t = times ? times[i] : 0.0;
        unsigned long long b = (unsigned long long)__double_as_longlong(t);
        b = (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);  // total order of doubles as unsigned
        key = b == ~0ull ? b - 1 : b;
        ok = 1;
      }
    }
    keys[i] = key;
    idx[i] = i;
  }
  unsigned m = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(count_out, __popc(m));
}
__global__ void k_gather_frame(int n_upper, const int* __restrict__ count, const int* __restrict__ idx_s, const double4* __restrict__ pts, const double* __restrict__ times, const double* __restrict__ intens, int global_shutter,
                               double4* __restrict__ o_pts, double* __restrict__ o_times, double* __restrict__ o_intens) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_upper || s >= *count) return;
  const int i = idx_s[s];
  o_pts[s] = pts[i];
  if (o_times) o_times[s] = (times && !global_shutter) ? times[i] : 0.0;
  if (intens && o_intens) o_intens[s] = intens[i];
}
__global__ void k_set_int(int* p, int v) { *p = v; }
__global__ void k_copy_last_pos(int n, const int* __restrict__ pos, int* __restrict__ out) { *out = n > 0 ? pos[n - 1] : 0; }

// covariance estimation (plane_covariance) writing the fp64 host-layout outputs and, when s0 is given, the fp32 planes of the
// device cloud in the caller's point order (the Morton reorder of gb_cloud_upload follows)
__global__ void __launch_bounds__(128) k_covariances_planes(int n_upper, const int* __restrict__ count, const double4* __restrict__ pts, const int* __restrict__ neighbors, int kc, int k,
                                                            double4* __restrict__ normals, double* __restrict__ covs, float4* __restrict__ s0, float4* __restrict__ s1, float* __restrict__ s2, float4* __restrict__ s3) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_upper || i >= *count) return;
  double C[9], nrm[3];
  const double4 p = plane_covariance(i, pts, neighbors, kc, k, C, nrm);
  const double nx = nrm[0], ny = nrm[1], nz = nrm[2];
  if (normals) normals[i] = make_double4(nx, ny, nz, 0.0);
  if (covs) store_cov4x4(covs + 16 * (size_t)i, C);
  if (!s0) return;
  // the host cast of PointCloudGPU::clone (fp64 -> fp32), upper triangle as gb_cloud_upload reads it from the column-major 4x4
  s0[i] = make_float4((float)p.x, (float)p.y, (float)p.z, (float)C[0]);
  s1[i] = make_float4((float)C[1], (float)C[2], (float)C[4], (float)C[5]);
  s2[i] = (float)C[8];
  s3[i] = make_float4((float)nx, (float)ny, (float)nz, 0.f);
}

// gb_cloud_estimate_covariances: the cloud's stored positions widened to fp64 (w = 1) in the caller's order (stored slot j
// holds the caller's point perm[j]), and the device count of them for the k-NN
__global__ void k_cloud_gather_points(int n, const float4* __restrict__ p0, const int* __restrict__ perm, double4* __restrict__ pts, int* __restrict__ count) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (j == 0) *count = n;
  const float4 a = p0[j];
  pts[perm ? perm[j] : j] = make_double4(a.x, a.y, a.z, 1.0);
}
// plane_covariance of the caller's point i (kc = k), cast once to fp32 as gb_cloud_upload casts it and stored into the cloud's
// slot inv_perm[i]: the covariance (p0.w, p1, p2) when p1 is given, the normal when normals is given.  Positions are not written.
__global__ void __launch_bounds__(128) k_cloud_covariances(int n, const double4* __restrict__ pts, const int* __restrict__ neighbors, int k, const int* __restrict__ inv_perm,
                                                           float4* __restrict__ p0, float4* __restrict__ p1, float* __restrict__ p2, float4* __restrict__ normals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double C[9], nrm[3];
  plane_covariance(i, pts, neighbors, k, k, C, nrm);
  const int o = inv_perm ? inv_perm[i] : i;
  if (p1) {
    p0[o].w = (float)C[0];
    p1[o] = make_float4((float)C[1], (float)C[2], (float)C[4], (float)C[5]);
    p2[o] = (float)C[8];
  }
  if (normals) normals[o] = make_float4((float)nrm[0], (float)nrm[1], (float)nrm[2], 0.f);
}

// ---- statistical outlier removal (cloud_preprocessor.cpp:165-167: gtsam_points::remove_outliers(frame, k, std_mul, threads)) [EXT]:
// d_i = mean distance of point i to its k nearest neighbours (the query itself included, as the k-NN returns it);
// keep i iff d_i < mean(d) + std_mul * sqrt(mean(d^2) - mean(d)^2)   (population variance over the frame) ----
__global__ void k_sor_dists(int n_upper, const int* __restrict__ count, const double4* __restrict__ pts, const int* __restrict__ nb, int k, double* __restrict__ dist, double* __restrict__ dist2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_upper) return;
  double d = 0.0;
  if (i < *count) {
    const double4 p = pts[i];
    double s = 0.0;
    for (int j = 0; j < k; j++) {
      const double4 q = pts[nb[(size_t)i * k + j]];
      const double ex = p.x - q.x, ey = p.y - q.y, ez = p.z - q.z;
      s += sqrt(__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez)));
    }
    d = s / k;
  }
  dist[i] = d;
  dist2[i] = __dmul_rn(d, d);
}
__global__ void k_sor_flags(int n_upper, const int* __restrict__ count, const double* __restrict__ dist, const double* __restrict__ sums /* [0] = sum d, [1] = sum d^2 */, double std_mul, int* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_upper) return;
  const int m = *count;
  const double mean = sums[0] / m;
  const double var = sums[1] / m - mean * mean;
  const double thresh = mean + std_mul * sqrt(var > 0.0 ? var : 0.0);
  keep[i] = (i < m && dist[i] < thresh) ? 1 : 0;
}
__global__ void k_sor_compact(int n_upper, const int* __restrict__ keep, const int* __restrict__ pos, const double4* __restrict__ pts, const double* __restrict__ times, const double* __restrict__ intens,
                              double4* __restrict__ o_pts, double* __restrict__ o_times, double* __restrict__ o_intens, int* __restrict__ count_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_upper) return;
  if (keep[i]) {
    const int o = pos[i] - 1;
    o_pts[o] = pts[i];
    o_times[o] = times[i];
    if (intens) o_intens[o] = intens[i];
  }
  if (i == n_upper - 1) *count_out = pos[i];
}

}  // namespace

gb_status gb_sor_dists(gb_ctx* ctx, int n, const int* d_count, const double4* pts, const int* nb, int k, double* dist, double* dist2) {
  return gb_launch(ctx, "k_sor_dists", k_sor_dists, (n + 255) / 256, 256, 0, n, d_count, pts, nb, k, dist, dist2);
}

gb_status gb_covariance_cloud(gb_ctx* ctx, int M, const int* d_count, const double4* pts, const int* neighbors, int kc, int k, double4* normals, double* covs,
                              const gb_planes& staged, const gb_sort_tmp& t, gb_cloud* cloud_out) {
  GB_CHECK(gb_launch(ctx, "k_covariances_planes", k_covariances_planes, (M + 127) / 128, 128, 0, M, d_count, pts, neighbors, kc, k, normals, covs, staged.p0, staged.p1, staged.p2,
                     staged.normals));
  if (cloud_out) GB_CHECK(gb_cloud_build(ctx, cloud_out, (size_t)M, staged, t));
  return GB_OK;
}

KnnTmp take_knn_tmp(Carver& cv, int n, void* cub, size_t cub_bytes) {
  KnnTmp t;
  t.ts = 1024;
  while (t.ts < 2u * (unsigned)n) t.ts <<= 1;
  t.s = gb_take_sort_tmp(cv, n, cub, cub_bytes);
  t.pts_s = cv.take<double4>(n);
  t.tables = cv.take<MlCell>((size_t)kMlLevels * t.ts);
  return t;
}

gb_status knn_device(gb_ctx* ctx, int n, const int* d_count, const double4* d_pts, int k, double h0, int* d_nb, const KnnTmp& t) {
  const int tb = 256, gb = (n + tb - 1) / tb;
  GB_CHECK(gb_launch(ctx, "k_fill_self", k_fill_self, (int)(((size_t)n * k + 255) / 256), 256, 0, n, k, d_nb));
  GB_CHECK(gb_launch(ctx, "k_ml_keys", k_ml_keys, gb, tb, 0, n, d_count, d_pts, 1.0 / h0, t.s.keys, t.s.idx));
  GB_CUB(ctx, cub::DeviceRadixSort::SortPairs, t.s.cub, t.s.cub_bytes, t.s.keys, t.s.keys_s, t.s.idx, t.s.idx_s, n, 0, 64);
  GB_CHECK(gb_launch(ctx, "k_ml_gather", k_ml_gather, gb, tb, 0, n, t.s.keys_s, t.s.idx_s, d_pts, t.pts_s));
  MlCell* tables = (MlCell*)t.tables;
  GB_CUDA(cudaMemsetAsync(tables, 0xff, sizeof(MlCell) * (size_t)kMlLevels * t.ts, ctx->stream));
  GB_CHECK(gb_launch(ctx, "k_ml_cells", k_ml_cells, gb, tb, 0, n, t.s.keys_s, tables, t.ts));
  return knn_dispatch(k, [&](auto K) {
    return gb_launch(ctx, "k_knn_pyramid", k_knn_pyramid<decltype(K)::value>, (n + 127) / 128, 128, 0, n, t.pts_s, t.s.keys_s, t.s.idx_s, tables, t.ts, 1.0 / h0, h0, d_nb);
  });
}

static gb_status preprocess(gb_ctx* ctx, size_t n_, const double* xyzw, const double* times, const double* intensities, const gb_preprocess_params* P, gb_preprocessed* out, gb_cloud* cloud_out) {
  const int n = (int)n_;
  cudaStream_t st = ctx->stream;
  const int k = P->k_correspondences;
  const size_t N = (size_t)n, cub_b = gb_cub_temp_bytes(N);
  gb_planes staged;  // fp32 planes of the device cloud, in frame order
  gb_sort_tmp t;
  KnnTmp knn;
  int *d_cnt, *d_flags, *d_pos, *d_starts, *d_keep, *d_nb, *d_nbo;
  double4 *d_raw, *d_ds, *d_fr, *d_nrm, *d_fr2;
  double *d_t, *d_i, *d_dst, *d_dsi, *d_frt, *d_fri, *d_cov, *d_dist, *d_dist2, *d_sums, *d_frt2, *d_fri2;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    staged = gb_cloud_planes(cv, N, true);
    void* d_cub = cv.take<char>(cub_b);
    t = gb_take_sort_tmp(cv, N, d_cub, cub_b);
    knn = take_knn_tmp(cv, n, d_cub, cub_b);
    d_cnt = cv.take<int>(64);  // [0] raw n, [1] after downsampling, [2] frame points, [3] voxels
    d_raw = cv.take<double4>(N);
    d_t = cv.take<double>(N);
    d_i = cv.take<double>(N);
    d_ds = cv.take<double4>(N);
    d_dst = cv.take<double>(N);
    d_dsi = cv.take<double>(N);
    d_fr = cv.take<double4>(N);
    d_frt = cv.take<double>(N);
    d_fri = cv.take<double>(N);
    d_flags = cv.take<int>(N + 1);
    d_pos = cv.take<int>(N + 1);
    d_starts = cv.take<int>(N + 1);
    d_keep = cv.take<int>(N + 1);
    d_nb = cv.take<int>(N * (size_t)k);
    d_nrm = cv.take<double4>(N);
    d_cov = cv.take<double>(16 * N);
    if (P->enable_outlier_removal) {
      d_nbo = cv.take<int>(N * (size_t)P->outlier_removal_k);
      d_dist = cv.take<double>(N);
      d_dist2 = cv.take<double>(N);
      d_sums = cv.take<double>(32);
      d_fr2 = cv.take<double4>(N);
      d_frt2 = cv.take<double>(N);
      d_fri2 = cv.take<double>(N);
    }
  }));
  const int tb = 256, gb = (n + tb - 1) / tb;

  GB_CHECK(gb_upload(ctx, {{d_raw, xyzw, sizeof(double4) * N}, {d_t, times, sizeof(double) * N}, {d_i, intensities, sizeof(double) * N}}));
  GB_CUDA(cudaMemsetAsync(d_cnt, 0, 256, st));
  GB_CHECK(gb_launch(ctx, "k_set_int", k_set_int, 1, 1, 0, d_cnt + 0, n));

  // ---- downsampling ----
  const double4* cur_pts = d_raw;
  const double* cur_t = times ? d_t : nullptr;
  const double* cur_i = intensities ? d_i : nullptr;
  const int* cur_cnt = d_cnt + 0;
  const int* keep = nullptr;
  if (P->downsample_resolution > 0.0) {
    GB_CHECK(gb_grid_keys(ctx, n, d_raw, 1.0 / P->downsample_resolution, nullptr, t.keys, t.idx));
    GB_CHECK(gb_group_by_key(ctx, n, t, d_flags, d_pos));
    GB_CHECK(gb_launch(ctx, "k_copy_last_pos", k_copy_last_pos, 1, 1, 0, n, d_pos, d_cnt + 3));  // V
    GB_CHECK(gb_group_starts(ctx, n, t, d_flags, d_pos, d_starts));
    if (P->use_random_grid_downsampling) {
      const double rate = P->downsample_target > 0 ? (double)P->downsample_target / (double)n : P->downsample_rate;  // :105
      if (rate < 0.99) {
        GB_CUDA(cudaMemsetAsync(d_keep, 0, sizeof(int) * N, st));
        GB_CHECK(gb_launch(ctx, "k_randomgrid_select", k_randomgrid_select, gb, tb, 0, n, d_cnt + 3, d_starts, t.idx_s, rate, P->seed, d_keep));
        const int cap = (int)((double)n * rate * 1.2);
        if (cap > 0 && cap < n)  // thin the survivors to 1.2 * rate * N: the smallest hashes stay
          GB_CHECK(gb_thin(ctx, n, d_keep, nullptr, cap, P->seed, t, d_keep));
        keep = d_keep;  // original order is kept; the gates below drop the rest
      }
    } else {
      GB_CHECK(gb_launch(ctx, "k_grid_means_counted", k_grid_means_counted, (n + 127) / 128, 128, 0, d_cnt + 3, d_starts, t.idx_s, d_raw, cur_t, cur_i, nullptr, d_ds, d_dst, d_dsi,
                         nullptr));
      cur_pts = d_ds; cur_t = times ? d_dst : nullptr; cur_i = intensities ? d_dsi : nullptr; cur_cnt = d_cnt + 3;
    }
  }
  // ---- gates + time order (one stable sort: rejected points sort to the end) ----
  FrameFilter ff;
  ff.near2 = P->distance_near_thresh * P->distance_near_thresh;
  ff.far2 = P->distance_far_thresh * P->distance_far_thresh;
  ff.crop = P->crop_bbox_frame;
  for (int a = 0; a < 3; a++) { ff.bmin[a] = P->crop_bbox_min[a]; ff.bmax[a] = P->crop_bbox_max[a]; }
  for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) ff.T[r * 4 + c] = P->T_imu_lidar[c * 4 + r];
  ff.global_shutter = P->global_shutter;
  GB_CHECK(gb_launch(ctx, "k_filter_time_keys", k_filter_time_keys, gb, tb, 0, n, cur_cnt, keep, cur_pts, cur_t, ff, t.keys, t.idx, d_cnt + 2));
  GB_CUB(ctx, cub::DeviceRadixSort::SortPairs, t.cub, cub_b, t.keys, t.keys_s, t.idx, t.idx_s, n, 0, 64);
  GB_CHECK(gb_launch(ctx, "k_gather_frame", k_gather_frame, gb, tb, 0, n, d_cnt + 2, t.idx_s, cur_pts, cur_t, cur_i, P->global_shutter, d_fr, d_frt, d_fri));
  const double h0 = P->knn_cell_size > 0.0 ? P->knn_cell_size : 0.25;
  const int* frame_cnt = d_cnt + 2;
  // ---- statistical outlier removal (optional) ----
  if (P->enable_outlier_removal) {
    const int ko = P->outlier_removal_k;
    GB_CHECK(knn_device(ctx, n, d_cnt + 2, d_fr, ko, h0, d_nbo, knn));
    GB_CHECK(gb_sor_dists(ctx, n, d_cnt + 2, d_fr, d_nbo, ko, d_dist, d_dist2));
    GB_CUB(ctx, cub::DeviceReduce::Sum, t.cub, cub_b, d_dist, d_sums, n);
    GB_CUB(ctx, cub::DeviceReduce::Sum, t.cub, cub_b, d_dist2, d_sums + 1, n);
    GB_CHECK(gb_launch(ctx, "k_sor_flags", k_sor_flags, gb, tb, 0, n, d_cnt + 2, d_dist, d_sums, P->outlier_std_mul_factor, d_keep));
    GB_CUB(ctx, cub::DeviceScan::InclusiveSum, t.cub, cub_b, d_keep, d_pos, n);
    GB_CHECK(gb_launch(ctx, "k_sor_compact", k_sor_compact, gb, tb, 0, n, d_keep, d_pos, d_fr, d_frt, intensities ? d_fri : nullptr, d_fr2, d_frt2, d_fri2, d_cnt + 4));
    d_fr = d_fr2; d_frt = d_frt2; d_fri = d_fri2;
    frame_cnt = d_cnt + 4;
  }
  // ---- k-NN ----
  GB_CHECK(knn_device(ctx, n, frame_cnt, d_fr, k, h0, d_nb, knn));
  // ---- the frame's point count (the one host synchronisation before the results) ----
  int M = 0;
  GB_CHECK(gb_download(ctx, {{&M, frame_cnt, sizeof(int)}}));
  out->num_points = (size_t)M;
  out->last_time = 0.0;
  if (M == 0) return GB_OK;
  // ---- covariances, written straight into the staged fp32 planes of the cloud (PointCloudGPU::clone on the device) ----
  if (P->estimate_covariances)  // the frame is gathered: t is free again
    GB_CHECK(gb_covariance_cloud(ctx, M, frame_cnt, d_fr, d_nb, k, P->k_neighbors_cov > 0 ? P->k_neighbors_cov : k, d_nrm, d_cov, staged, t, cloud_out));
  // ---- host products ----
  const size_t m = (size_t)M;
  const bool cov_out = P->estimate_covariances != 0;
  return gb_download(ctx, {{&out->last_time, d_frt + (M - 1), sizeof(double)}, {out->xyzw, d_fr, sizeof(double4) * m}, {out->times, d_frt, sizeof(double) * m},
                           {intensities ? out->intensities : nullptr, d_fri, sizeof(double) * m}, {out->neighbors, d_nb, sizeof(int) * m * (size_t)k},
                           {cov_out ? out->normals4 : nullptr, d_nrm, sizeof(double4) * m}, {cov_out ? out->cov4x4 : nullptr, d_cov, sizeof(double) * 16 * m}});
}

extern "C" gb_status gb_preprocess_default_params(gb_preprocess_params* p) {
  GB_REQUIRE(p, "null params");
  memset(p, 0, sizeof(*p));
  p->distance_near_thresh = 0.5;      // config_preprocess.json:20
  p->distance_far_thresh = 100.0;     // :21
  p->use_random_grid_downsampling = 1;  // :22
  p->downsample_resolution = 1.0;     // :23
  p->downsample_target = 10000;       // :24
  p->downsample_rate = 0.1;           // :25
  p->seed = 0;
  p->outlier_removal_k = 10;          // :27
  p->outlier_std_mul_factor = 1.0;    // :28
  p->k_correspondences = 10;          // :33
  p->estimate_covariances = 1;
  for (int i = 0; i < 4; i++) p->T_imu_lidar[i * 5] = 1.0;
  return GB_OK;
}
extern "C" gb_status gb_preprocess(gb_ctx* ctx, size_t n, const double* xyzw, const double* times, const double* intensities, const gb_preprocess_params* P, gb_preprocessed* out) {
  GB_REQUIRE(ctx && P && out, "null argument");
  out->num_points = 0; out->last_time = 0.0; out->cloud = nullptr;
  GB_REQUIRE(n < (size_t)1 << 30, "too many points");
  GB_REQUIRE(gb_knn_instantiated(P->k_correspondences), "k_correspondences is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_REQUIRE(P->k_neighbors_cov >= 0 && P->k_neighbors_cov <= P->k_correspondences, "k_neighbors_cov must be in [0, k_correspondences]");
  GB_REQUIRE(!P->enable_outlier_removal || gb_knn_instantiated(P->outlier_removal_k), "outlier_removal_k is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_REQUIRE(P->crop_bbox_frame >= 0 && P->crop_bbox_frame <= 2, "crop_bbox_frame must be 0 (off), 1 (lidar) or 2 (imu)");
  if (n == 0) return GB_OK;
  GB_REQUIRE(xyzw, "null points");
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(P->estimate_covariances ? new (std::nothrow) gb_cloud() : nullptr, cloud_free);
  if (P->estimate_covariances && !c) return GB_ERR_INTERNAL;
  if (c) { c->device = ctx->device; c->covs = true; }
  GB_CHECK(preprocess(ctx, n, xyzw, times, intensities, P, out, c.get()));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));  // the cloud is complete when the call returns (it may be used from another context)
  out->cloud = c.release();
  return GB_OK;
}

// knn_device with cell size 0.25 m on host arrays (the device-resident entry is inside gb_preprocess)
extern "C" gb_status gb_find_neighbors(gb_ctx* ctx, size_t n_, const double* xyzw, int k, int32_t* neighbors) {
  GB_REQUIRE(ctx, "null ctx");
  if (n_ == 0) return GB_OK;
  GB_REQUIRE(xyzw && neighbors && k > 0, "null argument");
  GB_REQUIRE(gb_knn_instantiated(k), "k is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_ENTER(ctx);
  const int n = (int)n_;
  const size_t N = (size_t)n, cub_b = gb_cub_temp_bytes(N);
  KnnTmp knn;
  int *d_cnt, *d_nb;
  double4* d_pts;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    knn = take_knn_tmp(cv, n, cv.take<char>(cub_b), cub_b);
    d_cnt = cv.take<int>(64);
    d_pts = cv.take<double4>(N);
    d_nb = cv.take<int>(N * (size_t)k);
  }));
  GB_CHECK(gb_upload(ctx, {{d_pts, xyzw, sizeof(double4) * N}}));
  GB_CHECK(gb_launch(ctx, "k_set_int", k_set_int, 1, 1, 0, d_cnt, n));
  GB_CHECK(knn_device(ctx, n, d_cnt, d_pts, k, 0.25, d_nb, knn));
  return gb_download(ctx, {{neighbors, d_nb, sizeof(int) * N * (size_t)k}});
}

// gb_find_neighbors and gb_covariances on a device cloud's own points, written back into its planes (the rule is in
// include/glim_b200.h): k_cloud_gather_points, knn_device at 0.25 m, k_cloud_covariances
extern "C" gb_status gb_cloud_estimate_covariances(gb_ctx* ctx, gb_cloud* cloud, int k_neighbors, int outputs) {
  GB_REQUIRE(ctx && cloud, "null argument");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(gb_knn_instantiated(k_neighbors), "k_neighbors is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)");
  GB_REQUIRE(outputs >= 1 && outputs <= (GB_CLOUD_COVARIANCES | GB_CLOUD_NORMALS), "outputs must be GB_CLOUD_COVARIANCES, GB_CLOUD_NORMALS or both");
  GB_REQUIRE(cloud->n * (size_t)k_neighbors < (size_t)1 << 30, "N * k_neighbors must be below 2^30");
  GB_ENTER(ctx);
  const bool covs = outputs & GB_CLOUD_COVARIANCES, normals = outputs & GB_CLOUD_NORMALS;
  if (normals) {  // the features were computed from the old normals: their block goes back to the pool here
    gb_dev_block old(ctx->device);
    old.hand_over(cloud->f_base);
    cloud->fpfh = nullptr;
  }
  const int n = (int)cloud->n, k = k_neighbors;
  if (n > 0) {
    gb_dev_block block(ctx->device);  // normals for a cloud built without them: a block of their own, handed over on success
    float4* d_normals = cloud->normals;
    if (normals && !d_normals) GB_CHECK(gb_dev_carve(ctx, block, [&](Carver& cv) { d_normals = cv.take<float4>((size_t)n); }));
    const size_t N = (size_t)n, cub_b = gb_cub_temp_bytes(N);
    KnnTmp knn;
    int *d_cnt, *d_nb;
    double4* d_pts;
    GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
      knn = take_knn_tmp(cv, n, cv.take<char>(cub_b), cub_b);
      d_cnt = cv.take<int>(1);
      d_pts = cv.take<double4>(N);
      d_nb = cv.take<int>(N * (size_t)k);
    }));
    GB_CHECK(gb_launch(ctx, "k_cloud_gather_points", k_cloud_gather_points, (n + 255) / 256, 256, 0, n, cloud->p0, cloud->perm, d_pts, d_cnt));
    GB_CHECK(knn_device(ctx, n, d_cnt, d_pts, k, 0.25, d_nb, knn));
    GB_CHECK(gb_launch(ctx, "k_cloud_covariances", k_cloud_covariances, (n + 127) / 128, 128, 0, n, d_pts, d_nb, k, cloud->inv_perm, cloud->p0, covs ? cloud->p1 : nullptr,
                       cloud->p2, normals ? d_normals : nullptr));
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (normals && !cloud->normals) {
      block.hand_over(cloud->n_base);
      cloud->normals = d_normals;
    }
  }
  if (covs) cloud->covs = true;
  return GB_OK;
}

// =============================================================================================
// gb_merge_frames: gtsam_points::merge_frames(poses, frames, downsample_resolution, target_num_points) as SubMapping calls it
// (src/glim/mapping/sub_mapping.cpp:481-497; the reference itself wanted merge_frames_gpu, commented out at :491): transform
// the keyframe clouds into the submap origin frame (points q = R p + t, covariances R C R^T), voxel-grid average points AND
// covariances at `downsample_resolution`, thin to `target_num_points` -- on the device, from the keyframes' device clouds.
// The averaging is fp64 in (frame, original point index) order: bit-exact with the oracle (go_merge_frames) on the same fp32
// inputs.  Thinning: the reference draws with std::mt19937; here the `target` voxels with the smallest hash(seed, voxel rank)
// stay, in key order ([EXT], unpinned).
// =============================================================================================
namespace {

__global__ void k_merge_transform(int num_frames, const gb_frame* __restrict__ frames, int total, double4* __restrict__ pts, double* __restrict__ cov6) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  const gb_frame& F = frames[gb_frame_of(frames, num_frames, g)];
  const int i = g - F.offset;
  const int slot = F.inv_perm ? F.inv_perm[i] : i;
  const float4 a0 = F.p0[slot];
  const float4 a1 = F.p1[slot];
  const float a2 = F.p2[slot];
  double q[3];
  gb_pose_record(F.T, a0, a1, a2, q, cov6 ? cov6 + 6 * (size_t)g : nullptr);
  pts[g] = make_double4(q[0], q[1], q[2], 1.0);
}
__global__ void k_merge_emit(int n_upper, const int* __restrict__ keep, const int* __restrict__ pos, const double4* __restrict__ pts, const double* __restrict__ cov6, double4* __restrict__ o_pts, double* __restrict__ o_cov16,
                             float4* __restrict__ s0, float4* __restrict__ s1, float* __restrict__ s2) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_upper || !keep[v]) return;
  const int o = pos[v] - 1;
  const double4 p = pts[v];
  const double* c = cov6 + 6 * (size_t)v;
  o_pts[o] = p;
  const double C[9] = {c[0], c[1], c[2], c[1], c[3], c[4], c[2], c[4], c[5]};
  store_cov4x4(o_cov16 + 16 * (size_t)o, C);
  s0[o] = make_float4((float)p.x, (float)p.y, (float)p.z, (float)c[0]);
  s1[o] = make_float4((float)c[1], (float)c[2], (float)c[3], (float)c[4]);
  s2[o] = (float)c[5];
}

}  // namespace

gb_status gb_frame_list_check(const gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, size_t* total) {
  GB_REQUIRE(K == 0 || (frames && poses), "null frames / poses");
  *total = 0;
  for (size_t k = 0; k < K; k++) {
    GB_REQUIRE(frames[k] && frames[k]->device == ctx->device, "null frame / frame on another device");
    GB_REQUIRE(frames[k]->n < ((size_t)1 << 32), "a frame of 2^32 points or more");
    *total += frames[k]->n;
  }
  GB_REQUIRE(*total < ((size_t)1 << 30), "too many points");
  return GB_OK;
}

bool gb_all_finite(const double* v, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (!std::isfinite(v[i])) return false;
  return true;
}

std::vector<gb_frame> gb_frame_table(size_t K, const gb_cloud* const* frames, const double* poses, const int* index) {
  std::vector<gb_frame> table(K);
  int offset = 0;
  for (size_t k = 0; k < K; k++) {
    const gb_cloud* c = frames[k];
    const double* T = poses + 16 * k;  // column-major 4x4
    gb_frame& F = table[k];
    F.p0 = c->p0; F.p1 = c->p1; F.p2 = c->p2; F.normals = c->normals; F.inv_perm = c->inv_perm;
    F.n = (int)c->n; F.offset = offset; F.index = index ? index[k] : (int)k;
    for (int r = 0; r < 3; r++) for (int cc = 0; cc < 4; cc++) F.T[r * 4 + cc] = T[cc * 4 + r];
    offset += F.n;
  }
  return table;
}

gb_status gb_transform_frames(gb_ctx* ctx, size_t K, const gb_frame* d_table, int total, double4* pts, double* cov6) {
  if (total == 0) return GB_OK;
  return gb_launch(ctx, "k_merge_transform", k_merge_transform, (total + 255) / 256, 256, 0, (int)K, d_table, total, pts, cov6);
}

static gb_status merge_frames(gb_ctx* ctx, int K, const gb_cloud* const* frames, const double* poses, double resolution, int target, unsigned long long seed, double* out_xyzw, double* out_cov4x4, size_t* num_out, gb_cloud* cloud_out) {
  cudaStream_t st = ctx->stream;
  size_t total = 0;
  for (int k = 0; k < K; k++) total += frames[k]->n;
  *num_out = 0;
  if (total == 0) return GB_OK;
  const int n = (int)total;
  const size_t N = total, cub_b = gb_cub_temp_bytes(N);
  const std::vector<gb_frame> table = gb_frame_table((size_t)K, frames, poses, nullptr);
  gb_planes staged;  // fp32 planes of the merged cloud, in output order
  gb_sort_tmp t;
  int *d_cnt, *d_flags, *d_pos, *d_starts, *d_keep;
  gb_frame* d_table;
  double4 *d_pts, *d_vpts;
  double *d_cov, *d_vcov, *d_ocov;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    staged = gb_cloud_planes(cv, N, false);
    t = gb_take_sort_tmp(cv, N, cv.take<char>(cub_b), cub_b);
    d_cnt = cv.take<int>(64);
    d_table = cv.take<gb_frame>(K);
    d_pts = cv.take<double4>(N);
    d_vpts = cv.take<double4>(N);
    d_cov = cv.take<double>(6 * N);
    d_vcov = cv.take<double>(6 * N);
    d_ocov = cv.take<double>(16 * N);
    d_flags = cv.take<int>(N + 1);
    d_pos = cv.take<int>(N + 1);
    d_starts = cv.take<int>(N + 1);
    d_keep = cv.take<int>(N + 1);
  }));
  GB_CUDA(cudaMemsetAsync(d_cnt, 0, 256, st));
  const int tb = 256, gb = (n + tb - 1) / tb;
  GB_CHECK(gb_upload(ctx, {{d_table, table.data(), sizeof(gb_frame) * K}}));
  GB_CHECK(gb_transform_frames(ctx, (size_t)K, d_table, n, d_pts, d_cov));
  GB_CHECK(gb_grid_keys(ctx, n, d_pts, 1.0 / resolution, nullptr, t.keys, t.idx));
  GB_CHECK(gb_group_by_key(ctx, n, t, d_flags, d_pos));
  GB_CHECK(gb_launch(ctx, "k_copy_last_pos", k_copy_last_pos, 1, 1, 0, n, d_pos, d_cnt));  // V
  GB_CHECK(gb_group_starts(ctx, n, t, d_flags, d_pos, d_starts));
  GB_CHECK(gb_launch(ctx, "k_grid_means_counted", k_grid_means_counted, (n + 127) / 128, 128, 0, d_cnt, d_starts, t.idx_s, d_pts, nullptr, nullptr, d_cov, d_vpts, nullptr,
                     nullptr, d_vcov));
  // keep flag per voxel v < V (all, or the `target` smallest hashes), then an inclusive scan gives the output slot
  GB_CHECK(gb_thin(ctx, n, nullptr, d_cnt, target, seed, t, d_keep));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, t.cub, cub_b, d_keep, d_pos, n);
  int M = 0;
  GB_CHECK(gb_download(ctx, {{&M, d_pos + (n - 1), sizeof(int)}}));
  *num_out = (size_t)M;
  if (M == 0) return GB_OK;
  GB_CHECK(gb_launch(ctx, "k_merge_emit", k_merge_emit, gb, tb, 0, n, d_keep, d_pos, d_vpts, d_vcov, d_pts /* reused: emitted points */, d_ocov, staged.p0, staged.p1, staged.p2));
  if (cloud_out) GB_CHECK(gb_cloud_build(ctx, cloud_out, (size_t)M, staged, t));
  return gb_download(ctx, {{out_xyzw, d_pts, sizeof(double4) * (size_t)M}, {out_cov4x4, d_ocov, sizeof(double) * 16 * (size_t)M}});
}

extern "C" gb_status gb_merge_frames(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, double resolution, int target, uint64_t seed, double* out_xyzw, double* out_cov4x4, size_t* num_out, gb_cloud** out_cloud) {
  GB_REQUIRE(ctx && num_out, "null argument");
  *num_out = 0;
  if (out_cloud) *out_cloud = nullptr;
  if (K == 0) return GB_OK;
  GB_REQUIRE(resolution > 0.0, "downsample_resolution must be positive");
  size_t total = 0;
  GB_CHECK(gb_frame_list_check(ctx, K, frames, poses, &total));  // poses may be non-finite: their points get no voxel key
  GB_REQUIRE(K < 65536, "too many frames");
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(out_cloud ? new (std::nothrow) gb_cloud() : nullptr, cloud_free);
  if (out_cloud && !c) return GB_ERR_INTERNAL;
  if (c) { c->device = ctx->device; c->covs = true; }
  GB_CHECK(merge_frames(ctx, (int)K, frames, poses, resolution, target, seed, out_xyzw, out_cov4x4, num_out, c.get()));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (out_cloud) *out_cloud = c.release();
  return GB_OK;
}

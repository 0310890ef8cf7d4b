// gb_kernels_preprocess.cu -- per-frame preprocess on the GPU (sm_90a): k-NN, covariance / normal
// estimation, voxel-grid downsampling.
//
// Replaces, at GLIM's call sites:
//   CloudPreprocessor::find_neighbors            src/glim/preprocess/cloud_preprocessor.cpp:190-221  (gtsam_points::KdTree::knn_search)
//   CloudCovarianceEstimation::estimate (PLANE)  src/glim/common/cloud_covariance_estimation.cpp:43-122, :181-196
//   gtsam_points::voxelgrid_sampling             src/glim/preprocess/cloud_preprocessor.cpp:108
// Oracles: go_knn_bruteforce, go_covariance_estimate, go_voxelgrid_sampling (oracle/glim_oracle.c).
// All three work in fp64 like the reference's host code (Vector4d / Matrix4d).
#include "gb_internal.cuh"

#include <cub/cub.cuh>
#include <cmath>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

namespace {

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------
// exact k-NN, brute force over shared-memory tiles.  One query per thread, candidates streamed
// in ascending index with a strict '<' insertion, so ties resolve to the lower index exactly as
// in the oracle.  The query itself is a candidate (distance 0), as in the reference (:196).
// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(128) k_knn_bruteforce(int n, const double4* __restrict__ pts, int* __restrict__ neighbors) {
  constexpr int TILE = 256;
  __shared__ double sx[TILE], sy[TILE], sz[TILE];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double px = 0, py = 0, pz = 0;
  if (i < n) { const double4 p = pts[i]; px = p.x; py = p.y; pz = p.z; }
  double bd[K];
  int bi[K];
#pragma unroll
  for (int k = 0; k < K; k++) { bd[k] = 1e300; bi[k] = i; }
  int cnt = 0;
  for (int base = 0; base < n; base += TILE) {
    __syncthreads();
    for (int t = threadIdx.x; t < TILE; t += blockDim.x) {
      const int j = base + t;
      if (j < n) { const double4 q = pts[j]; sx[t] = q.x; sy[t] = q.y; sz[t] = q.z; }
    }
    __syncthreads();
    const int m = min(TILE, n - base);
    if (i < n) {
      for (int t = 0; t < m; t++) {
        const double dx = px - sx[t], dy = py - sy[t], dz = pz - sz[t];
        // no FMA contraction: bit-identical to the oracle's (dx*dx + dy*dy) + dz*dz
        const double d = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (d < bd[K - 1]) {
          // insert (d, base+t) keeping ascending distance; equal distances stay behind earlier ones
          double cd = d;
          int ci = base + t;
#pragma unroll
          for (int k = 0; k < K; k++) {
            if (cd < bd[k]) {
              const double td = bd[k]; const int ti = bi[k];
              bd[k] = cd; bi[k] = ci; cd = td; ci = ti;
            }
          }
          cnt++;
        }
      }
    }
  }
  if (i < n) {
    const int found = min(cnt, K);
#pragma unroll
    for (int k = 0; k < K; k++) neighbors[(size_t)i * K + k] = k < found ? bi[k] : i;
  }
}

// ---------------------------------------------------------------------------------------------
// exact k-NN on a uniform grid.  Points are sorted by the packed key of their cell (x major, z minor), so the cells of one
// (x, y) column with consecutive z are one contiguous key range: a ring of the search cube costs (2r+1)^2 binary searches.
// One query per thread, in sorted order (spatially coherent warps).  After ring r every unseen point lies outside the cube
// of cells [c-r, c+r]^3, i.e. at least m*h away (m = distance from the query to the nearest cube face, in cells), so the
// search stops as soon as the k-th best distance is within that bound -- the result is EXACT, with the same
// (distance, index) tie rule and the same un-contracted fp64 distance as the brute-force kernel and the oracle.
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kKnnInvalid = ~0ull;

__global__ void k_knn_keys(int n, const double4* __restrict__ pts, double inv_h, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double4 p = pts[i];
  unsigned long long key = kKnnInvalid;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    const double fx = floor(p.x * inv_h), fy = floor(p.y * inv_h), fz = floor(p.z * inv_h);
    if (fabs(fx) < 1048575.0 && fabs(fy) < 1048575.0 && fabs(fz) < 1048575.0) {
      unsigned long long k;
      if (gb_pack_key((int)fx, (int)fy, (int)fz, &k)) key = k;
    }
  }
  keys[i] = key;
  idx[i] = i;
}
__global__ void k_knn_gather(int n, const int* __restrict__ idx_s, const double4* __restrict__ pts, double4* __restrict__ pts_s) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) pts_s[s] = pts[idx_s[s]];
}
__global__ void k_count_heads(int n, const unsigned long long* __restrict__ keys_s, int* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int head = 0;
  if (i < n) { const unsigned long long k = keys_s[i]; head = (k != kKnnInvalid && (i == 0 || keys_s[i - 1] != k)) ? 1 : 0; }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) head += __shfl_xor_sync(0xffffffffu, head, o);
  if ((threadIdx.x & 31) == 0 && head) atomicAdd(count, head);
}

__device__ __forceinline__ int knn_lower_bound(const unsigned long long* __restrict__ keys, int n, unsigned long long key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(&keys[mid]) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

template <int K>
__global__ void __launch_bounds__(128) k_knn_grid(int n, const double4* __restrict__ pts_s, const unsigned long long* __restrict__ keys_s, const int* __restrict__ idx_s,
                                                  double inv_h, double h, int3 cmin, int3 cmax, int max_ring, int* __restrict__ neighbors) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int self = idx_s[t];
  const unsigned long long key = keys_s[t];
  double bd[K];
  int bi[K];
#pragma unroll
  for (int k = 0; k < K; k++) { bd[k] = 1e300; bi[k] = 0x7fffffff; }
  int cnt = 0;
  if (key != kKnnInvalid) {
    const double4 p = pts_s[t];
    int cx, cy, cz;
    gb_unpack_key(key, cx, cy, cz);
    const double ux = p.x * inv_h - (double)cx, uy = p.y * inv_h - (double)cy, uz = p.z * inv_h - (double)cz;  // in [0, 1)
    // the cube must eventually cover every occupied cell
    const int rmax = max(max(max(cx - cmin.x, cmax.x - cx), max(cy - cmin.y, cmax.y - cy)), max(cz - cmin.z, cmax.z - cz));
    // ring r costs (2r+1)^2 range searches: an isolated point (a far return with no neighbours nearby) would walk thousands of
    // empty rings.  After max_ring rings (chosen on the host so that the ring walk costs about as much as one pass over all
    // points) without a proof of completeness the query falls back to a scan of ALL points (exact, O(N)).
    bool complete = false;
    for (int r = 0; r <= min(rmax, max_ring); r++) {
      for (int dx = -r; dx <= r; dx++) {
        const int x = cx + dx;
        if (x < cmin.x || x > cmax.x) continue;
        for (int dy = -r; dy <= r; dy++) {
          const int y = cy + dy;
          if (y < cmin.y || y > cmax.y) continue;
          const bool edge = (abs(dx) == r) || (abs(dy) == r);
          // edge columns contribute their whole z range; interior columns only the two new cells at z = cz -+ r
          const int nseg = edge ? 1 : 2;
          for (int sgi = 0; sgi < nseg; sgi++) {
            int z0, z1;
            if (edge) { z0 = cz - r; z1 = cz + r; } else { z0 = z1 = (sgi == 0) ? cz - r : cz + r; }
            z0 = max(z0, cmin.z); z1 = min(z1, cmax.z);
            if (z0 > z1) continue;
            unsigned long long klo, khi;
            gb_pack_key(x, y, z0, &klo);
            gb_pack_key(x, y, z1, &khi);
            for (int s = knn_lower_bound(keys_s, n, klo); s < n; s++) {
              if (__ldg(&keys_s[s]) > khi) break;
              const double4 q = pts_s[s];
              const double ex = p.x - q.x, ey = p.y - q.y, ez = p.z - q.z;
              const double d = __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
              const int j = __ldg(&idx_s[s]);
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
          }
        }
      }
      if (r == rmax) { complete = true; break; }  // the cube covers every occupied cell
      if (cnt >= K) {
        const double m = fmin(fmin(fmin(ux, 1.0 - ux), fmin(uy, 1.0 - uy)), fmin(uz, 1.0 - uz)) + (double)r;
        const double bound = m * h * (1.0 - 1e-12);
        if (bd[K - 1] <= bound * bound) { complete = true; break; }
      }
    }
    if (!complete) {
#pragma unroll
      for (int k = 0; k < K; k++) { bd[k] = 1e300; bi[k] = 0x7fffffff; }
      cnt = 0;
      for (int s = 0; s < n; s++) {
        if (__ldg(&keys_s[s]) == kKnnInvalid) break;  // invalid points sort last
        const double4 q = pts_s[s];
        const double ex = p.x - q.x, ey = p.y - q.y, ez = p.z - q.z;
        const double d = __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
        const int j = __ldg(&idx_s[s]);
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
    }
  }
  const int found = min(cnt, K);
#pragma unroll
  for (int k = 0; k < K; k++) neighbors[(size_t)self * K + k] = k < found ? bi[k] : self;
}

// ---------------------------------------------------------------------------------------------
// closed-form symmetric 3x3 eigen decomposition (same published algorithm as the oracle's
// go_eigen_sym3_direct / Eigen's computeDirect): evals ascending, V[r*3+k] = k-th eigenvector.
// ---------------------------------------------------------------------------------------------
__device__ inline void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ inline void extract_kernel(const double* m, double* res, double* rep) {
  int i0 = 0;
  double best = fabs(m[0]);
  if (fabs(m[4]) > best) { best = fabs(m[4]); i0 = 1; }
  if (fabs(m[8]) > best) { best = fabs(m[8]); i0 = 2; }
  double c1v[3], c2v[3];
  const int i1 = (i0 + 1) % 3, i2 = (i0 + 2) % 3;
  for (int r = 0; r < 3; r++) { rep[r] = m[r * 3 + i0]; c1v[r] = m[r * 3 + i1]; c2v[r] = m[r * 3 + i2]; }
  double c0[3], c1[3];
  cross3(rep, c1v, c0);
  cross3(rep, c2v, c1);
  const double n0 = c0[0] * c0[0] + c0[1] * c0[1] + c0[2] * c0[2];
  const double n1 = c1[0] * c1[0] + c1[1] * c1[1] + c1[2] * c1[2];
  if (n0 > n1) { const double s = 1.0 / sqrt(n0); for (int k = 0; k < 3; k++) res[k] = c0[k] * s; }
  else if (n1 > 0.0) { const double s = 1.0 / sqrt(n1); for (int k = 0; k < 3; k++) res[k] = c1[k] * s; }
  else { res[0] = 1; res[1] = 0; res[2] = 0; }
}
__device__ void eigen_sym3_direct(const double* A, double* evals, double* V) {
  const double shift = (A[0] + A[4] + A[8]) / 3.0;
  double m[9];
  for (int k = 0; k < 9; k++) m[k] = A[k];
  m[0] -= shift; m[4] -= shift; m[8] -= shift;
  double scale = 0.0;
  for (int k = 0; k < 9; k++) scale = fmax(scale, fabs(m[k]));
  if (scale > 0.0) for (int k = 0; k < 9; k++) m[k] /= scale;
  const double m00 = m[0], m11 = m[4], m22 = m[8], m10 = m[3], m20 = m[6], m21 = m[7];
  const double c0 = m00 * m11 * m22 + 2.0 * m10 * m20 * m21 - m00 * m21 * m21 - m11 * m20 * m20 - m22 * m10 * m10;
  const double c1 = m00 * m11 - m10 * m10 + m00 * m22 - m20 * m20 + m11 * m22 - m21 * m21;
  const double c2 = m00 + m11 + m22;
  const double c2_3 = c2 / 3.0;
  double a_3 = (c2 * c2_3 - c1) / 3.0;
  if (a_3 < 0.0) a_3 = 0.0;
  const double half_b = 0.5 * (c0 + c2_3 * (2.0 * c2_3 * c2_3 - c1));
  double qq = a_3 * a_3 * a_3 - half_b * half_b;
  if (qq < 0.0) qq = 0.0;
  const double rho = sqrt(a_3);
  const double theta = atan2(sqrt(qq), half_b) / 3.0;
  const double ct = cos(theta), st = sin(theta);
  const double s3 = 1.7320508075688772935;
  double ev[3];
  ev[0] = c2_3 - rho * (ct + s3 * st);
  ev[1] = c2_3 - rho * (ct - s3 * st);
  ev[2] = c2_3 + 2.0 * rho * ct;
  const double eps = 2.220446049250313e-16;
  if ((ev[2] - ev[0]) <= eps) {
    for (int k = 0; k < 9; k++) V[k] = 0.0;
    V[0] = V[4] = V[8] = 1.0;
  } else {
    double d0 = ev[2] - ev[1], d1 = ev[1] - ev[0];
    int k = 0, l = 2;
    if (d0 > d1) { const double t = d0; d0 = d1; d1 = t; k = 2; l = 0; }
    double tmp[9], vk[3], vl[3], rep[3];
    for (int e = 0; e < 9; e++) tmp[e] = m[e];
    tmp[0] -= ev[k]; tmp[4] -= ev[k]; tmp[8] -= ev[k];
    extract_kernel(tmp, vk, rep);
    if (d0 <= 2.0 * eps * d1) {
      const double dp = vk[0] * rep[0] + vk[1] * rep[1] + vk[2] * rep[2];
      for (int r = 0; r < 3; r++) vl[r] = rep[r] - dp * vk[r];
      const double nl = sqrt(vl[0] * vl[0] + vl[1] * vl[1] + vl[2] * vl[2]);
      if (nl > 0) for (int r = 0; r < 3; r++) vl[r] /= nl;
    } else {
      double dummy[3];
      for (int e = 0; e < 9; e++) tmp[e] = m[e];
      tmp[0] -= ev[l]; tmp[4] -= ev[l]; tmp[8] -= ev[l];
      extract_kernel(tmp, vl, dummy);
    }
    double v0[3], v1[3], v2[3];
    for (int r = 0; r < 3; r++) { v0[r] = (k == 0) ? vk[r] : vl[r]; v2[r] = (k == 0) ? vl[r] : vk[r]; }
    cross3(v2, v0, v1);
    const double n1 = sqrt(v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2]);
    if (n1 > 0) for (int r = 0; r < 3; r++) v1[r] /= n1;
    for (int r = 0; r < 3; r++) { V[r * 3 + 0] = v0[r]; V[r * 3 + 1] = v1[r]; V[r * 3 + 2] = v2[r]; }
  }
  for (int k = 0; k < 3; k++) evals[k] = ev[k] * scale + shift;
}

// CloudCovarianceEstimation::estimate, calc_cov (cloud_covariance_estimation.cpp:80-102).
// The reference materialises pt_cross = p p^T per point (:58-63) and gathers 128-byte rows; here the
// outer products are formed in registers from the gathered neighbour points (same sums, same order).
__global__ void __launch_bounds__(128) k_covariances(int n, const double4* __restrict__ pts, const int* __restrict__ neighbors, int kc, int k, double4* __restrict__ normals, double* __restrict__ covs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double S[4] = {0, 0, 0, 0};
  double X[16];
  for (int e = 0; e < 16; e++) X[e] = 0.0;
  const size_t begin = (size_t)kc * (size_t)i;
  for (int j = 0; j < k; j++) {
    const double4 q = pts[neighbors[begin + j]];
    const double p[4] = {q.x, q.y, q.z, q.w};
    for (int r = 0; r < 4; r++) S[r] += p[r];
    for (int c = 0; c < 4; c++)
      for (int r = 0; r < 4; r++) X[c * 4 + r] += p[r] * p[c];
  }
  double mean[4], A[9];
  for (int r = 0; r < 4; r++) mean[r] = S[r] / k;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) A[r * 3 + c] = (X[c * 4 + r] - mean[r] * S[c]) / k;
  double evals[3], V[9];
  eigen_sym3_direct(A, evals, V);
  const double values[3] = {1e-3, 1.0, 1.0};
  double* C = covs + 16 * (size_t)i;
  for (int e = 0; e < 16; e++) C[e] = 0.0;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double s = 0;
      for (int e = 0; e < 3; e++) s += V[r * 3 + e] * values[e] * V[c * 3 + e];
      C[c * 4 + r] = s;
    }
  const double4 p = pts[i];
  double nx = V[0], ny = V[3], nz = V[6];
  if (p.x * nx + p.y * ny + p.z * nz > 0.0) { nx = -nx; ny = -ny; nz = -nz; }
  normals[i] = make_double4(nx, ny, nz, 0.0);
}

// ---------------------------------------------------------------------------------------------
// voxel-grid downsampling (fp64 coordinates, SURVEY C.2)
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kInvalidKey = ~0ull;

__global__ void k_grid_keys(int n, const double4* __restrict__ pts, double inv_res, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double4 p = pts[i];
  unsigned long long key = kInvalidKey;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    const double fx = floor(p.x * inv_res), fy = floor(p.y * inv_res), fz = floor(p.z * inv_res);
    if (fabs(fx) < 2e9 && fabs(fy) < 2e9 && fabs(fz) < 2e9) {
      unsigned long long k;
      if (gb_pack_key((int)fx, (int)fy, (int)fz, &k)) key = k;
    }
  }
  keys[i] = key;
  idx[i] = i;
}
__global__ void k_grid_flags(int n, const unsigned long long* __restrict__ keys, int* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  flags[i] = (k != kInvalidKey && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
}
__global__ void k_grid_starts(int n, const unsigned long long* __restrict__ keys, const int* __restrict__ flags, const int* __restrict__ pos, int* __restrict__ starts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flags[i]) starts[pos[i] - 1] = i;
  const bool valid = keys[i] != kInvalidKey;
  const bool next_valid = (i + 1 < n) && keys[i + 1] != kInvalidKey;
  if (valid && !next_valid) starts[pos[i]] = i + 1;
}
__global__ void k_grid_means(int V, const int* __restrict__ starts, const int* __restrict__ idx, const double4* __restrict__ pts, const double* __restrict__ times, const double* __restrict__ intens,
                             double4* __restrict__ out_pts, double* __restrict__ out_times, double* __restrict__ out_intens) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int b = starts[v], e = starts[v + 1];
  double sx = 0, sy = 0, sz = 0, sw = 0, st = 0, si = 0;
  for (int s = b; s < e; s++) {
    const int i = idx[s];
    const double4 p = pts[i];
    sx += p.x; sy += p.y; sz += p.z; sw += p.w;
    if (times) st += times[i];
    if (intens) si += intens[i];
  }
  const int cnt = e - b;
  out_pts[v] = make_double4(sx / cnt, sy / cnt, sz / cnt, sw / cnt);
  if (times) out_times[v] = st / cnt;
  if (intens) out_intens[v] = si / cnt;
}

}  // namespace

template <int K>
static void launch_knn(bool grid, int n, const double4* d_pts, const double4* d_pts_s, const unsigned long long* d_keys_s, const int* d_idx_s, double inv_h, double h, int3 cmin, int3 cmax, int* d_nb, cudaStream_t st) {
  const int tb = 128, gb = (n + tb - 1) / tb;
  // (4/3) R^3 range searches of log2(n) steps each ~ n  =>  R = cbrt(0.75 n / log2 n)
  const int max_ring = std::min(64, std::max(6, (int)cbrt(0.75 * (double)n / std::max(1.0, log2((double)n)))));
  if (grid) k_knn_grid<K><<<gb, tb, 0, st>>>(n, d_pts_s, d_keys_s, d_idx_s, inv_h, h, cmin, cmax, max_ring, d_nb);
  else k_knn_bruteforce<K><<<gb, tb, 0, st>>>(n, d_pts, d_nb);
}

gb_status gb_find_neighbors_impl(gb_ctx* ctx, size_t n_, const double* xyzw, int k, int32_t* neighbors) {
  const int n = (int)n_;
  if (n == 0) return GB_OK;
  cudaStream_t st = ctx->stream;
  const char* mode = getenv("GB_KNN");
  const bool grid = mode ? (strcmp(mode, "grid") == 0) : (n >= 4096);
  size_t cub_sort = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
  const size_t pts_b = align_up(sizeof(double4) * (size_t)n, 256), nb_b = align_up(sizeof(int) * (size_t)n * k, 256);
  const size_t key_b = align_up(sizeof(unsigned long long) * (size_t)n, 256), idx_b = align_up(sizeof(int) * (size_t)n, 256), cub_b = align_up(cub_sort, 256);
  char* base = nullptr;
  GB_CHECK(gb_ctx_scratch(ctx, 2 * pts_b + nb_b + 2 * key_b + 2 * idx_b + cub_b + 256, (void**)&base));
  char* p = base;
  double4* d_pts = (double4*)p; p += pts_b;
  double4* d_pts_s = (double4*)p; p += pts_b;
  int* d_nb = (int*)p; p += nb_b;
  unsigned long long* d_keys = (unsigned long long*)p; p += key_b;
  unsigned long long* d_keys_s = (unsigned long long*)p; p += key_b;
  int* d_idx = (int*)p; p += idx_b;
  int* d_idx_s = (int*)p; p += idx_b;
  void* d_cub = p; p += cub_b;
  int* d_count = (int*)p;
  GB_CUDA(cudaMemcpyAsync(d_pts, xyzw, sizeof(double4) * (size_t)n, cudaMemcpyHostToDevice, st));
  double h = 0.25, inv_h = 4.0;
  int3 cmin = make_int3(0, 0, 0), cmax = make_int3(0, 0, 0);
  if (grid) {
    const int tb = 256, gb = (n + tb - 1) / tb;
    // cell size: measure the occupancy at 0.25 m, then aim for ~4 points per occupied cell (points lie on surfaces:
    // points per cell grows with h^2); a second pass re-sorts at the chosen size
    for (int pass = 0; pass < 2; pass++) {
      inv_h = 1.0 / h;
      k_knn_keys<<<gb, tb, 0, st>>>(n, d_pts, inv_h, d_keys, d_idx);
      size_t tmp = cub_b;
      GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, d_idx_s, n, 0, 64, st));
      ctx->launches += 2;
      if (pass == 1) break;
      int occ = 0;
      GB_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int), st));
      k_count_heads<<<gb, tb, 0, st>>>(n, d_keys_s, d_count);
      GB_CUDA(cudaMemcpyAsync(&occ, d_count, sizeof(int), cudaMemcpyDeviceToHost, st));
      GB_CUDA(cudaStreamSynchronize(st));
      ctx->launches++;
      const double per_cell = occ > 0 ? (double)n / occ : 1.0;
      double h2 = h * sqrt(4.0 / per_cell);
      h2 = fmin(4.0, fmax(0.02, h2));
      if (fabs(h2 - h) < 0.1 * h) break;  // close enough: keep the first sort
      h = h2;
    }
    inv_h = 1.0 / h;
    k_knn_gather<<<gb, tb, 0, st>>>(n, d_idx_s, d_pts, d_pts_s);
    ctx->launches++;
    // bounding box of the occupied cells (host: one pass over the caller's array, same floor(p * inv_h) as the kernel)
    bool any = false;
    for (int i = 0; i < n; i++) {
      const double* q = xyzw + 4 * (size_t)i;
      if (!(std::isfinite(q[0]) && std::isfinite(q[1]) && std::isfinite(q[2]))) continue;
      const double fx = floor(q[0] * inv_h), fy = floor(q[1] * inv_h), fz = floor(q[2] * inv_h);
      if (!(fabs(fx) < 1048575.0 && fabs(fy) < 1048575.0 && fabs(fz) < 1048575.0)) continue;
      const int x = (int)fx, y = (int)fy, z = (int)fz;
      if (!any) { cmin = cmax = make_int3(x, y, z); any = true; }
      cmin.x = std::min(cmin.x, x); cmin.y = std::min(cmin.y, y); cmin.z = std::min(cmin.z, z);
      cmax.x = std::max(cmax.x, x); cmax.y = std::max(cmax.y, y); cmax.z = std::max(cmax.z, z);
    }
  }
  switch (k) {
#define GB_KNN_CASE(K) case K: launch_knn<K>(grid, n, d_pts, d_pts_s, d_keys_s, d_idx_s, inv_h, h, cmin, cmax, d_nb, st); break;
    GB_KNN_CASE(1) GB_KNN_CASE(2) GB_KNN_CASE(3) GB_KNN_CASE(4) GB_KNN_CASE(5) GB_KNN_CASE(6) GB_KNN_CASE(7) GB_KNN_CASE(8)
    GB_KNN_CASE(9) GB_KNN_CASE(10) GB_KNN_CASE(12) GB_KNN_CASE(15) GB_KNN_CASE(16) GB_KNN_CASE(20) GB_KNN_CASE(24) GB_KNN_CASE(32)
#undef GB_KNN_CASE
    default:
      gb_set_error("k = %d is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)", k);
      return GB_ERR_INVALID_ARGUMENT;
  }
  GB_CUDA(cudaGetLastError());
  ctx->launches++;
  GB_CUDA(cudaMemcpyAsync(neighbors, d_nb, sizeof(int) * (size_t)n * k, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return GB_OK;
}

gb_status gb_covariances_impl(gb_ctx* ctx, size_t n_, const double* xyzw, const int32_t* neighbors, int kc, int k, double* normals4, double* cov4x4) {
  const int n = (int)n_;
  if (n == 0) return GB_OK;  // cloud_covariance_estimation.cpp:49-51
  cudaStream_t st = ctx->stream;
  const size_t pts_b = align_up(sizeof(double4) * (size_t)n, 256), nb_b = align_up(sizeof(int) * (size_t)n * kc, 256);
  const size_t nrm_b = pts_b, cov_b = align_up(sizeof(double) * 16 * (size_t)n, 256);
  char* base = nullptr;
  GB_CHECK(gb_ctx_scratch(ctx, pts_b + nb_b + nrm_b + cov_b, (void**)&base));
  double4* d_pts = (double4*)base;
  int* d_nb = (int*)(base + pts_b);
  double4* d_nrm = (double4*)(base + pts_b + nb_b);
  double* d_cov = (double*)(base + pts_b + nb_b + nrm_b);
  GB_CUDA(cudaMemcpyAsync(d_pts, xyzw, sizeof(double4) * (size_t)n, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_nb, neighbors, sizeof(int) * (size_t)n * kc, cudaMemcpyHostToDevice, st));
  k_covariances<<<(n + 127) / 128, 128, 0, st>>>(n, d_pts, d_nb, kc, k, d_nrm, d_cov);
  GB_CUDA(cudaGetLastError());
  ctx->launches++;
  GB_CUDA(cudaMemcpyAsync(normals4, d_nrm, sizeof(double4) * (size_t)n, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaMemcpyAsync(cov4x4, d_cov, sizeof(double) * 16 * (size_t)n, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return GB_OK;
}

gb_status gb_voxelgrid_sampling_impl(gb_ctx* ctx, size_t n_, const double* xyzw, const double* times, const double* intensities, double resolution, double* out_xyzw, double* out_times, double* out_intensities, size_t* num_out) {
  const int n = (int)n_;
  *num_out = 0;
  if (n == 0) return GB_OK;
  cudaStream_t st = ctx->stream;
  size_t cub_sort = 0, cub_scan = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
  cub::DeviceScan::InclusiveSum(nullptr, cub_scan, (int*)nullptr, (int*)nullptr, n, st);
  const size_t cub_b = align_up(cub_sort > cub_scan ? cub_sort : cub_scan, 256);
  const size_t pts_b = align_up(sizeof(double4) * (size_t)n, 256), d_b = align_up(sizeof(double) * (size_t)n, 256);
  const size_t key_b = align_up(sizeof(unsigned long long) * (size_t)n, 256), i_b = align_up(sizeof(int) * (size_t)(n + 1), 256);
  char* base = nullptr;
  GB_CHECK(gb_ctx_scratch(ctx, cub_b + 2 * pts_b + 4 * d_b + 2 * key_b + 5 * i_b, (void**)&base));
  char* p = base;
  void* d_cub = p; p += cub_b;
  double4* d_pts = (double4*)p; p += pts_b;
  double4* d_opts = (double4*)p; p += pts_b;
  double* d_t = (double*)p; p += d_b;
  double* d_i = (double*)p; p += d_b;
  double* d_ot = (double*)p; p += d_b;
  double* d_oi = (double*)p; p += d_b;
  unsigned long long* d_keys = (unsigned long long*)p; p += key_b;
  unsigned long long* d_keys_s = (unsigned long long*)p; p += key_b;
  int* d_idx = (int*)p; p += i_b;
  int* d_idx_s = (int*)p; p += i_b;
  int* d_flags = (int*)p; p += i_b;
  int* d_pos = (int*)p; p += i_b;
  int* d_starts = (int*)p; p += i_b;
  GB_CUDA(cudaMemcpyAsync(d_pts, xyzw, sizeof(double4) * (size_t)n, cudaMemcpyHostToDevice, st));
  if (times) GB_CUDA(cudaMemcpyAsync(d_t, times, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, st));
  if (intensities) GB_CUDA(cudaMemcpyAsync(d_i, intensities, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, st));
  const int tb = 256, gb = (n + tb - 1) / tb;
  k_grid_keys<<<gb, tb, 0, st>>>(n, d_pts, 1.0 / resolution, d_keys, d_idx);
  size_t tmp = cub_b;
  GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, d_idx_s, n, 0, 64, st));
  k_grid_flags<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags);
  tmp = cub_b;
  GB_CUDA(cub::DeviceScan::InclusiveSum(d_cub, tmp, d_flags, d_pos, n, st));
  int V = 0;
  GB_CUDA(cudaMemcpyAsync(&V, d_pos + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  ctx->launches += 4;
  if (V > 0) {
    k_grid_starts<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags, d_pos, d_starts);
    k_grid_means<<<(V + 127) / 128, 128, 0, st>>>(V, d_starts, d_idx_s, d_pts, times ? d_t : nullptr, intensities ? d_i : nullptr, d_opts, d_ot, d_oi);
    GB_CUDA(cudaGetLastError());
    ctx->launches += 2;
    GB_CUDA(cudaMemcpyAsync(out_xyzw, d_opts, sizeof(double4) * (size_t)V, cudaMemcpyDeviceToHost, st));
    if (times && out_times) GB_CUDA(cudaMemcpyAsync(out_times, d_ot, sizeof(double) * (size_t)V, cudaMemcpyDeviceToHost, st));
    if (intensities && out_intensities) GB_CUDA(cudaMemcpyAsync(out_intensities, d_oi, sizeof(double) * (size_t)V, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
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
__device__ __forceinline__ unsigned long long spread21(unsigned long long x) {
  x &= 0x1fffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}
__device__ __forceinline__ unsigned long long morton3(unsigned x, unsigned y, unsigned z) { return (spread21(x) << 2) | (spread21(y) << 1) | spread21(z); }

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
// scans all points.  Same un-contracted fp64 distance and (distance, index) tie rule as the brute-force kernel and the oracle.
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
// C.2); here it is the ppv points with the smallest hash(seed, index) -- a fixed pseudo-random choice the oracle shares.
__device__ __forceinline__ unsigned long long rg_hash(unsigned long long seed, unsigned i) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1u);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
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

__global__ void k_rg_hash_keys(int n, const int* __restrict__ keep, unsigned long long seed, unsigned long long* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = keep[i] ? rg_hash(seed, (unsigned)i) : ~0ull;
}
__global__ void k_rg_cap(int n, int cap, const unsigned long long* __restrict__ sorted, unsigned long long seed, int* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && keep[i] && rg_hash(seed, (unsigned)i) > sorted[cap - 1]) keep[i] = 0;
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
__global__ void k_grid_means_counted(const int* __restrict__ num_voxels, const int* __restrict__ starts, const int* __restrict__ idx, const double4* __restrict__ pts, const double* __restrict__ times, const double* __restrict__ intens,
                                     double4* __restrict__ out_pts, double* __restrict__ out_times, double* __restrict__ out_intens) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= *num_voxels) return;
  const int b = starts[v], e = starts[v + 1];
  double sx = 0, sy = 0, sz = 0, sw = 0, st = 0, si = 0;
  for (int s = b; s < e; s++) {  // same sums in the same order as k_grid_means / the oracle
    const int i = idx[s];
    const double4 p = pts[i];
    sx += p.x; sy += p.y; sz += p.z; sw += p.w;
    if (times) st += times[i];
    if (intens) si += intens[i];
  }
  const int cnt = e - b;
  out_pts[v] = make_double4(sx / cnt, sy / cnt, sz / cnt, sw / cnt);
  if (times) out_times[v] = st / cnt;
  if (intens) out_intens[v] = si / cnt;
}
__global__ void k_set_int(int* p, int v) { *p = v; }
__global__ void k_copy_last_pos(int n, const int* __restrict__ pos, int* __restrict__ out) { *out = n > 0 ? pos[n - 1] : 0; }

// covariance estimation (same arithmetic as k_covariances) writing the fp64 host-layout outputs AND the fp32 planes of the
// device cloud in the caller's point order (the Morton reorder of gb_cloud_upload follows)
__global__ void __launch_bounds__(128) k_covariances_planes(int n_upper, const int* __restrict__ count, const double4* __restrict__ pts, const int* __restrict__ neighbors, int kc, int k,
                                                            double4* __restrict__ normals, double* __restrict__ covs, float4* __restrict__ s0, float4* __restrict__ s1, float* __restrict__ s2, float4* __restrict__ s3) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_upper || i >= *count) return;
  double S[4] = {0, 0, 0, 0};
  double X[16];
  for (int e = 0; e < 16; e++) X[e] = 0.0;
  const size_t begin = (size_t)kc * (size_t)i;
  for (int j = 0; j < k; j++) {
    const double4 q = pts[neighbors[begin + j]];
    const double p[4] = {q.x, q.y, q.z, q.w};
    for (int r = 0; r < 4; r++) S[r] += p[r];
    for (int c = 0; c < 4; c++)
      for (int r = 0; r < 4; r++) X[c * 4 + r] += p[r] * p[c];
  }
  double mean[4], A[9];
  for (int r = 0; r < 4; r++) mean[r] = S[r] / k;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) A[r * 3 + c] = (X[c * 4 + r] - mean[r] * S[c]) / k;
  double evals[3], V[9];
  eigen_sym3_direct(A, evals, V);
  const double values[3] = {1e-3, 1.0, 1.0};
  double C[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double s = 0;
      for (int e = 0; e < 3; e++) s += V[r * 3 + e] * values[e] * V[c * 3 + e];
      C[r * 3 + c] = s;
    }
  const double4 p = pts[i];
  double nx = V[0], ny = V[3], nz = V[6];
  if (p.x * nx + p.y * ny + p.z * nz > 0.0) { nx = -nx; ny = -ny; nz = -nz; }
  if (normals) normals[i] = make_double4(nx, ny, nz, 0.0);
  if (covs) {
    double* Co = covs + 16 * (size_t)i;
    for (int e = 0; e < 16; e++) Co[e] = 0.0;
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) Co[c * 4 + r] = C[r * 3 + c];
  }
  // the host cast of PointCloudGPU::clone (fp64 -> fp32), upper triangle as gb_cloud_upload reads it from the column-major 4x4
  s0[i] = make_float4((float)p.x, (float)p.y, (float)p.z, (float)C[0]);
  s1[i] = make_float4((float)C[1], (float)C[2], (float)C[4], (float)C[5]);
  s2[i] = (float)C[8];
  s3[i] = make_float4((float)nx, (float)ny, (float)nz, 0.f);
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

template <int K>
static void launch_knn_pyramid(int n, const double4* pts_s, const unsigned long long* keys_s, const int* idx_s, const MlCell* tables, unsigned ts, double inv_h0, double h0, int* nb, cudaStream_t st) {
  k_knn_pyramid<K><<<(n + 127) / 128, 128, 0, st>>>(n, pts_s, keys_s, idx_s, tables, ts, inv_h0, h0, nb);
}

}  // namespace

// scratch carving
struct Carver {
  char* base; size_t off;
  template <typename T> T* take(size_t count) { T* p = (T*)(base + off); off += align_up(sizeof(T) * count, 256); return p; }
};

// exact k-NN of the first *d_count points of d_pts (device resident); neighbors[i * k + j]
static gb_status knn_device(gb_ctx* ctx, int n, const int* d_count, const double4* d_pts, int k, double h0, int* d_nb, Carver& cv, size_t cub_b, void* d_cub) {
  cudaStream_t st = ctx->stream;
  unsigned ts = 1024;
  while (ts < 2u * (unsigned)n) ts <<= 1;
  unsigned long long* keys = cv.take<unsigned long long>(n);
  unsigned long long* keys_s = cv.take<unsigned long long>(n);
  int* idx = cv.take<int>(n);
  int* idx_s = cv.take<int>(n);
  double4* pts_s = cv.take<double4>(n);
  MlCell* tables = cv.take<MlCell>((size_t)kMlLevels * ts);
  const int tb = 256, gb = (n + tb - 1) / tb;
  k_fill_self<<<(int)(((size_t)n * k + 255) / 256), 256, 0, st>>>(n, k, d_nb);
  k_ml_keys<<<gb, tb, 0, st>>>(n, d_count, d_pts, 1.0 / h0, keys, idx);
  size_t tmp = cub_b;
  GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, keys, keys_s, idx, idx_s, n, 0, 64, st));
  k_ml_gather<<<gb, tb, 0, st>>>(n, keys_s, idx_s, d_pts, pts_s);
  GB_CUDA(cudaMemsetAsync(tables, 0xff, sizeof(MlCell) * (size_t)kMlLevels * ts, st));
  k_ml_cells<<<gb, tb, 0, st>>>(n, keys_s, tables, ts);
  switch (k) {
#define GB_KNN_CASE(K) case K: launch_knn_pyramid<K>(n, pts_s, keys_s, idx_s, tables, ts, 1.0 / h0, h0, d_nb, st); break;
    GB_KNN_CASE(1) GB_KNN_CASE(2) GB_KNN_CASE(3) GB_KNN_CASE(4) GB_KNN_CASE(5) GB_KNN_CASE(6) GB_KNN_CASE(7) GB_KNN_CASE(8)
    GB_KNN_CASE(9) GB_KNN_CASE(10) GB_KNN_CASE(12) GB_KNN_CASE(15) GB_KNN_CASE(16) GB_KNN_CASE(20) GB_KNN_CASE(24) GB_KNN_CASE(32)
#undef GB_KNN_CASE
    default:
      gb_set_error("k = %d is not an instantiated neighbour count (1-10, 12, 15, 16, 20, 24, 32)", k);
      return GB_ERR_INVALID_ARGUMENT;
  }
  GB_CUDA(cudaGetLastError());
  ctx->launches += 6;
  return GB_OK;
}

gb_status gb_preprocess_impl(gb_ctx* ctx, size_t n_, const double* xyzw, const double* times, const double* intensities, const gb_preprocess_params* P, gb_preprocessed* out, gb_cloud* cloud_out) {
  const int n = (int)n_;
  cudaStream_t st = ctx->stream;
  const int k = P->k_correspondences;
  size_t cub_sort = 0, cub_scan = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
  cub::DeviceScan::InclusiveSum(nullptr, cub_scan, (int*)nullptr, (int*)nullptr, n, st);
  size_t cub_keys = 0, cub_red = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_keys, (unsigned long long*)nullptr, (unsigned long long*)nullptr, n, 0, 64, st);
  cub::DeviceReduce::Sum(nullptr, cub_red, (double*)nullptr, (double*)nullptr, n, st);
  const size_t cub_b = align_up(std::max(std::max(std::max(cub_sort, cub_scan), cub_keys), cub_red), 256);
  unsigned ts = 1024;
  while (ts < 2u * (unsigned)n) ts <<= 1;
  const size_t N = (size_t)n;
  const size_t planes = 2 * align_up(16 * N, 256) + align_up(4 * N, 256) + align_up(16 * N, 256);
  const size_t total = cub_b + 256 /*counters*/ + 3 * align_up(32 * N, 256) /*raw, ds, frame pts*/ + 6 * align_up(8 * N, 256) /*times, intens x3*/ + 4 * align_up(8 * N, 256) /*keys x2 (+2 knn)*/
                       + 8 * align_up(4 * (N + 1), 256) /*idx, flags, pos, starts, keep ...*/ + align_up(4 * N * (size_t)k, 256) + align_up(32 * N, 256) /*normals*/ + align_up(128 * N, 256) /*covs*/
                       + align_up(32 * N, 256) /*knn pts_s*/ + align_up(sizeof(MlCell) * (size_t)kMlLevels * ts, 256) + gb_cloud_reorder_scratch_bytes(N, planes) + 4096
                       + (P->enable_outlier_removal ? align_up(4 * N * (size_t)std::max(1, P->outlier_removal_k), 256) + 4 * align_up(8 * N, 256) + align_up(32 * N, 256) + 256  /* SOR arrays */
                                                          + 2 * align_up(8 * N, 256) + 2 * align_up(4 * N, 256) + align_up(32 * N, 256) + align_up(sizeof(MlCell) * (size_t)kMlLevels * ts, 256) /* second k-NN */ : 0);
  char* base = nullptr;
  GB_CHECK(gb_ctx_scratch(ctx, total, (void**)&base));
  Carver cv{base, 0};
  // the staged planes + the reorder's temporaries come first (gb_cloud_reorder_impl expects its temporaries behind the planes)
  char* staged = cv.take<char>(gb_cloud_reorder_scratch_bytes(N, planes));
  void* d_cub = cv.take<char>(cub_b);
  int* d_cnt = cv.take<int>(64);  // [0] raw n, [1] after downsampling, [2] frame points, [3] voxels
  double4* d_raw = cv.take<double4>(N);
  double* d_t = cv.take<double>(N);
  double* d_i = cv.take<double>(N);
  double4* d_ds = cv.take<double4>(N);
  double* d_dst = cv.take<double>(N);
  double* d_dsi = cv.take<double>(N);
  double4* d_fr = cv.take<double4>(N);
  double* d_frt = cv.take<double>(N);
  double* d_fri = cv.take<double>(N);
  unsigned long long* d_keys = cv.take<unsigned long long>(N);
  unsigned long long* d_keys_s = cv.take<unsigned long long>(N);
  int* d_idx = cv.take<int>(N + 1);
  int* d_idx_s = cv.take<int>(N + 1);
  int* d_flags = cv.take<int>(N + 1);
  int* d_pos = cv.take<int>(N + 1);
  int* d_starts = cv.take<int>(N + 1);
  int* d_keep = cv.take<int>(N + 1);
  int* d_nb = cv.take<int>(N * (size_t)k);
  double4* d_nrm = cv.take<double4>(N);
  double* d_cov = cv.take<double>(16 * N);
  const int tb = 256, gb = (n + tb - 1) / tb;

  GB_CUDA(cudaMemcpyAsync(d_raw, xyzw, sizeof(double4) * N, cudaMemcpyHostToDevice, st));
  if (times) GB_CUDA(cudaMemcpyAsync(d_t, times, sizeof(double) * N, cudaMemcpyHostToDevice, st));
  if (intensities) GB_CUDA(cudaMemcpyAsync(d_i, intensities, sizeof(double) * N, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemsetAsync(d_cnt, 0, 256, st));
  k_set_int<<<1, 1, 0, st>>>(d_cnt + 0, n);

  // ---- downsampling ----
  const double4* cur_pts = d_raw;
  const double* cur_t = times ? d_t : nullptr;
  const double* cur_i = intensities ? d_i : nullptr;
  const int* cur_cnt = d_cnt + 0;
  const int* keep = nullptr;
  if (P->downsample_resolution > 0.0) {
    k_grid_keys<<<gb, tb, 0, st>>>(n, d_raw, 1.0 / P->downsample_resolution, d_keys, d_idx);
    size_t tmp = cub_b;
    GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, d_idx_s, n, 0, 64, st));
    k_grid_flags<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags);
    tmp = cub_b;
    GB_CUDA(cub::DeviceScan::InclusiveSum(d_cub, tmp, d_flags, d_pos, n, st));
    k_copy_last_pos<<<1, 1, 0, st>>>(n, d_pos, d_cnt + 3);  // V
    k_grid_starts<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags, d_pos, d_starts);
    ctx->launches += 5;
    if (P->use_random_grid_downsampling) {
      const double rate = P->downsample_target > 0 ? (double)P->downsample_target / (double)n : P->downsample_rate;  // :105
      if (rate < 0.99) {
        GB_CUDA(cudaMemsetAsync(d_keep, 0, sizeof(int) * N, st));
        k_randomgrid_select<<<gb, tb, 0, st>>>(n, d_cnt + 3, d_starts, d_idx_s, rate, P->seed, d_keep);
        const int cap = (int)((double)n * rate * 1.2);
        if (cap > 0 && cap < n) {  // thin the survivors to 1.2 * rate * N: the smallest hashes stay
          k_rg_hash_keys<<<gb, tb, 0, st>>>(n, d_keep, P->seed, d_keys);
          size_t tmp2 = cub_b;
          GB_CUDA(cub::DeviceRadixSort::SortKeys(d_cub, tmp2, d_keys, d_keys_s, n, 0, 64, st));
          k_rg_cap<<<gb, tb, 0, st>>>(n, cap, d_keys_s, P->seed, d_keep);
          ctx->launches += 3;
        }
        ctx->launches++;
        keep = d_keep;  // original order is kept; the gates below drop the rest
      }
    } else {
      k_grid_means_counted<<<(n + 127) / 128, 128, 0, st>>>(d_cnt + 3, d_starts, d_idx_s, d_raw, cur_t, cur_i, d_ds, d_dst, d_dsi);
      ctx->launches++;
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
  k_filter_time_keys<<<gb, tb, 0, st>>>(n, cur_cnt, keep, cur_pts, cur_t, ff, d_keys, d_idx, d_cnt + 2);
  {
    size_t tmp = cub_b;
    GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, d_idx_s, n, 0, 64, st));
  }
  k_gather_frame<<<gb, tb, 0, st>>>(n, d_cnt + 2, d_idx_s, cur_pts, cur_t, cur_i, P->global_shutter, d_fr, d_frt, d_fri);
  ctx->launches += 3;
  const double h0 = P->knn_cell_size > 0.0 ? P->knn_cell_size : 0.25;
  const int* frame_cnt = d_cnt + 2;
  // ---- statistical outlier removal (optional) ----
  if (P->enable_outlier_removal) {
    const int ko = P->outlier_removal_k;
    int* d_nbo = cv.take<int>(N * (size_t)ko);
    double* d_dist = cv.take<double>(N);
    double* d_dist2 = cv.take<double>(N);
    double* d_sums = cv.take<double>(32);
    double4* d_fr2 = cv.take<double4>(N);
    double* d_frt2 = cv.take<double>(N);
    double* d_fri2 = cv.take<double>(N);
    GB_CHECK(knn_device(ctx, n, d_cnt + 2, d_fr, ko, h0, d_nbo, cv, cub_b, d_cub));
    k_sor_dists<<<gb, tb, 0, st>>>(n, d_cnt + 2, d_fr, d_nbo, ko, d_dist, d_dist2);
    size_t tmp = cub_b;
    GB_CUDA(cub::DeviceReduce::Sum(d_cub, tmp, d_dist, d_sums, n, st));
    tmp = cub_b;
    GB_CUDA(cub::DeviceReduce::Sum(d_cub, tmp, d_dist2, d_sums + 1, n, st));
    k_sor_flags<<<gb, tb, 0, st>>>(n, d_cnt + 2, d_dist, d_sums, P->outlier_std_mul_factor, d_keep);
    tmp = cub_b;
    GB_CUDA(cub::DeviceScan::InclusiveSum(d_cub, tmp, d_keep, d_pos, n, st));
    k_sor_compact<<<gb, tb, 0, st>>>(n, d_keep, d_pos, d_fr, d_frt, intensities ? d_fri : nullptr, d_fr2, d_frt2, d_fri2, d_cnt + 4);
    ctx->launches += 6;
    d_fr = d_fr2; d_frt = d_frt2; d_fri = d_fri2;
    frame_cnt = d_cnt + 4;
  }
  // ---- k-NN ----
  GB_CHECK(knn_device(ctx, n, frame_cnt, d_fr, k, h0, d_nb, cv, cub_b, d_cub));
  // ---- the frame's point count (the one host synchronisation before the results) ----
  int M = 0;
  GB_CUDA(cudaMemcpyAsync(&M, frame_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  out->num_points = (size_t)M;
  // ---- covariances, written straight into the staged fp32 planes of the cloud (PointCloudGPU::clone on the device) ----
  if (P->estimate_covariances && M > 0) {
    const size_t c0 = align_up(16 * (size_t)M, 256), c2 = align_up(4 * (size_t)M, 256);
    float4* s0 = (float4*)staged;
    float4* s1 = (float4*)(staged + c0);
    float* s2 = (float*)(staged + 2 * c0);
    float4* s3 = (float4*)(staged + 2 * c0 + c2);
    k_covariances_planes<<<(M + 127) / 128, 128, 0, st>>>(M, frame_cnt, d_fr, d_nb, k, P->k_neighbors_cov > 0 ? P->k_neighbors_cov : k, d_nrm, d_cov, s0, s1, s2, s3);
    GB_CUDA(cudaGetLastError());
    ctx->launches++;
    if (cloud_out) {
      const size_t ctotal = 3 * c0 + c2;
      const size_t bperm = align_up(sizeof(int) * (size_t)M, 256);
      cloud_out->n = (size_t)M;
      GB_CUDA(gb_dev_malloc(ctx->device, ctotal + 2 * bperm, &cloud_out->base));
      cloud_out->bytes = ctotal + 2 * bperm;
      char* d = (char*)cloud_out->base;
      cloud_out->p0 = (float4*)d; cloud_out->p1 = (float4*)(d + c0); cloud_out->p2 = (float*)(d + 2 * c0); cloud_out->normals = (float4*)(d + 2 * c0 + c2);
      cloud_out->perm = (int*)(d + ctotal); cloud_out->inv_perm = (int*)(d + ctotal + bperm);
      GB_CHECK(gb_cloud_reorder_impl(ctx, cloud_out, staged, c0, c0, c2, c0));
    }
  }
  // ---- host products: D2H into the context's pinned staging (full PCIe rate), then one memcpy each into the caller's arrays ----
  if (M > 0) {
    const size_t m = (size_t)M;
    const bool cov_out = P->estimate_covariances != 0;
    struct Part { void* dst; const void* src; size_t bytes; };
    Part parts[6] = {{out->xyzw, d_fr, sizeof(double4) * m}, {out->times, d_frt, sizeof(double) * m}, {(out->intensities && intensities) ? out->intensities : nullptr, d_fri, sizeof(double) * m},
                     {out->neighbors, d_nb, sizeof(int) * m * (size_t)k}, {(cov_out ? out->normals4 : nullptr), d_nrm, sizeof(double4) * m}, {(cov_out ? out->cov4x4 : nullptr), d_cov, sizeof(double) * 16 * m}};
    size_t total_h = 64;
    for (const Part& q : parts) if (q.dst) total_h += align_up(q.bytes, 64);
    char* h = nullptr;
    GB_CHECK(gb_ctx_pinned(ctx, total_h, (void**)&h));
    size_t off = 64;
    GB_CUDA(cudaMemcpyAsync(h, d_frt + (M - 1), sizeof(double), cudaMemcpyDeviceToHost, st));
    for (const Part& q : parts) {
      if (!q.dst) continue;
      GB_CUDA(cudaMemcpyAsync(h + off, q.src, q.bytes, cudaMemcpyDeviceToHost, st));
      off += align_up(q.bytes, 64);
    }
    GB_CUDA(cudaStreamSynchronize(st));
    memcpy(&out->last_time, h, sizeof(double));
    off = 64;
    for (const Part& q : parts) {
      if (!q.dst) continue;
      memcpy(q.dst, h + off, q.bytes);
      off += align_up(q.bytes, 64);
    }
  } else {
    out->last_time = 0.0;
  }
  return GB_OK;
}

// gb_find_neighbors on the pyramid (host arrays in / out; the device-resident entry is inside gb_preprocess)
gb_status gb_find_neighbors_pyramid_impl(gb_ctx* ctx, size_t n_, const double* xyzw, int k, int32_t* neighbors) {
  const int n = (int)n_;
  cudaStream_t st = ctx->stream;
  size_t cub_sort = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
  const size_t cub_b = align_up(cub_sort, 256), N = (size_t)n;
  unsigned ts = 1024;
  while (ts < 2u * (unsigned)n) ts <<= 1;
  const size_t total = cub_b + 256 + 2 * align_up(32 * N, 256) + 2 * align_up(8 * N, 256) + 2 * align_up(4 * N, 256) + align_up(4 * N * (size_t)k, 256) + align_up(sizeof(MlCell) * (size_t)kMlLevels * ts, 256) + 4096;
  char* base = nullptr;
  GB_CHECK(gb_ctx_scratch(ctx, total, (void**)&base));
  Carver cv{base, 0};
  void* d_cub = cv.take<char>(cub_b);
  int* d_cnt = cv.take<int>(64);
  double4* d_pts = cv.take<double4>(N);
  int* d_nb = cv.take<int>(N * (size_t)k);
  GB_CUDA(cudaMemcpyAsync(d_pts, xyzw, sizeof(double4) * N, cudaMemcpyHostToDevice, st));
  k_set_int<<<1, 1, 0, st>>>(d_cnt, n);
  GB_CHECK(knn_device(ctx, n, d_cnt, d_pts, k, 0.25, d_nb, cv, cub_b, d_cub));
  GB_CUDA(cudaMemcpyAsync(neighbors, d_nb, sizeof(int) * N * (size_t)k, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
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

struct MergeFrame { const float4* p0; const float4* p1; const float* p2; const int* inv_perm; int n; int offset; double T[12]; };

__global__ void k_merge_transform(int num_frames, const MergeFrame* __restrict__ frames, int total, double4* __restrict__ pts, double* __restrict__ cov6) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  int f = 0;
  while (f + 1 < num_frames && frames[f + 1].offset <= g) f++;
  const MergeFrame& F = frames[f];
  const int i = g - F.offset;
  const int slot = F.inv_perm ? F.inv_perm[i] : i;
  const float4 a0 = F.p0[slot];
  const float4 a1 = F.p1[slot];
  const float a2 = F.p2[slot];
  const double* T = F.T;  // rows of the 3x4 pose
  // un-contracted fp64 with a fixed association order: bit-exact with the oracle (go_merge_frames, built with fp-contract=off)
  const double x = a0.x, y = a0.y, z = a0.z;
  double q[3];
  for (int r = 0; r < 3; r++) q[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[r * 4 + 0], x), __dmul_rn(T[r * 4 + 1], y)), __dmul_rn(T[r * 4 + 2], z)), T[r * 4 + 3]);
  pts[g] = make_double4(q[0], q[1], q[2], 1.0);
  const double C[9] = {a0.w, a1.x, a1.y, a1.x, a1.z, a1.w, a1.y, a1.w, a2};
  double RC[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) RC[r * 3 + c] = __dadd_rn(__dadd_rn(__dmul_rn(T[r * 4 + 0], C[0 * 3 + c]), __dmul_rn(T[r * 4 + 1], C[1 * 3 + c])), __dmul_rn(T[r * 4 + 2], C[2 * 3 + c]));
  double* o = cov6 + 6 * (size_t)g;
  int e = 0;
  for (int r = 0; r < 3; r++)
    for (int c = r; c < 3; c++) o[e++] = __dadd_rn(__dadd_rn(__dmul_rn(RC[r * 3 + 0], T[c * 4 + 0]), __dmul_rn(RC[r * 3 + 1], T[c * 4 + 1])), __dmul_rn(RC[r * 3 + 2], T[c * 4 + 2]));
}
__global__ void k_merge_means(const int* __restrict__ num_voxels, const int* __restrict__ starts, const int* __restrict__ idx, const double4* __restrict__ pts, const double* __restrict__ cov6,
                              double4* __restrict__ o_pts, double* __restrict__ o_cov6) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= *num_voxels) return;
  const int b = starts[v], e = starts[v + 1];
  double s[4] = {0, 0, 0, 0}, c[6] = {0, 0, 0, 0, 0, 0};
  for (int k = b; k < e; k++) {
    const int i = idx[k];
    const double4 p = pts[i];
    s[0] += p.x; s[1] += p.y; s[2] += p.z; s[3] += p.w;
    for (int m = 0; m < 6; m++) c[m] += cov6[6 * (size_t)i + m];
  }
  const int cnt = e - b;
  o_pts[v] = make_double4(s[0] / cnt, s[1] / cnt, s[2] / cnt, s[3] / cnt);
  for (int m = 0; m < 6; m++) o_cov6[6 * (size_t)v + m] = c[m] / cnt;
}
__global__ void k_merge_hash_keys(int n_upper, const int* __restrict__ num_voxels, unsigned long long seed, unsigned long long* __restrict__ keys) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n_upper) keys[v] = v < *num_voxels ? rg_hash(seed, (unsigned)v) : ~0ull;
}
// keep flag per voxel (all, or the `target` smallest hashes), then an inclusive scan gives the output slot
__global__ void k_merge_keep(int n_upper, const int* __restrict__ num_voxels, int target, const unsigned long long* __restrict__ sorted, unsigned long long seed, int* __restrict__ keep) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_upper) return;
  int k = v < *num_voxels;
  if (k && target > 0 && target < *num_voxels) k = rg_hash(seed, (unsigned)v) <= sorted[target - 1];
  keep[v] = k;
}
__global__ void k_merge_emit(int n_upper, const int* __restrict__ keep, const int* __restrict__ pos, const double4* __restrict__ pts, const double* __restrict__ cov6, double4* __restrict__ o_pts, double* __restrict__ o_cov16,
                             float4* __restrict__ s0, float4* __restrict__ s1, float* __restrict__ s2) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_upper || !keep[v]) return;
  const int o = pos[v] - 1;
  const double4 p = pts[v];
  const double* c = cov6 + 6 * (size_t)v;
  o_pts[o] = p;
  double* C = o_cov16 + 16 * (size_t)o;
  for (int e = 0; e < 16; e++) C[e] = 0.0;
  C[0] = c[0]; C[4] = c[1]; C[8] = c[2]; C[1] = c[1]; C[5] = c[3]; C[9] = c[4]; C[2] = c[2]; C[6] = c[4]; C[10] = c[5];
  s0[o] = make_float4((float)p.x, (float)p.y, (float)p.z, (float)c[0]);
  s1[o] = make_float4((float)c[1], (float)c[2], (float)c[3], (float)c[4]);
  s2[o] = (float)c[5];
}

}  // namespace

gb_status gb_merge_frames_impl(gb_ctx* ctx, int K, const gb_cloud* const* frames, const double* poses, double resolution, int target, unsigned long long seed, double* out_xyzw, double* out_cov4x4, size_t* num_out, gb_cloud* cloud_out) {
  cudaStream_t st = ctx->stream;
  size_t total = 0;
  std::vector<MergeFrame> mf((size_t)K);
  for (int k = 0; k < K; k++) {
    const gb_cloud* c = frames[k];
    MergeFrame& F = mf[(size_t)k];
    F.p0 = c->p0; F.p1 = c->p1; F.p2 = c->p2; F.inv_perm = c->inv_perm; F.n = (int)c->n; F.offset = (int)total;
    for (int r = 0; r < 3; r++) for (int cc = 0; cc < 4; cc++) F.T[r * 4 + cc] = poses[(size_t)k * 16 + cc * 4 + r];
    total += c->n;
  }
  *num_out = 0;
  if (total == 0) return GB_OK;
  const int n = (int)total;
  const size_t N = total;
  size_t cub_sort = 0, cub_scan = 0, cub_keys = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n, 0, 64, st);
  cub::DeviceScan::InclusiveSum(nullptr, cub_scan, (int*)nullptr, (int*)nullptr, n, st);
  cub::DeviceRadixSort::SortKeys(nullptr, cub_keys, (unsigned long long*)nullptr, (unsigned long long*)nullptr, n, 0, 64, st);
  const size_t cub_b = align_up(std::max(std::max(cub_sort, cub_scan), cub_keys), 256);
  const size_t planes = 2 * align_up(16 * N, 256) + align_up(4 * N, 256);
  const size_t need = gb_cloud_reorder_scratch_bytes(N, planes) + cub_b + 256 + align_up(sizeof(MergeFrame) * (size_t)K, 256) + 2 * align_up(32 * N, 256) + 2 * align_up(48 * N, 256) + align_up(128 * N, 256)
                      + 2 * align_up(8 * N, 256) + 6 * align_up(4 * (N + 1), 256) + 4096;
  char* base = nullptr;
  GB_CHECK(gb_ctx_scratch(ctx, need, (void**)&base));
  Carver cv{base, 0};
  char* staged = cv.take<char>(gb_cloud_reorder_scratch_bytes(N, planes));
  void* d_cub = cv.take<char>(cub_b);
  int* d_cnt = cv.take<int>(64);
  MergeFrame* d_mf = cv.take<MergeFrame>((size_t)K);
  double4* d_pts = cv.take<double4>(N);
  double4* d_vpts = cv.take<double4>(N);
  double* d_cov = cv.take<double>(6 * N);
  double* d_vcov = cv.take<double>(6 * N);
  double* d_ocov = cv.take<double>(16 * N);
  unsigned long long* d_keys = cv.take<unsigned long long>(N);
  unsigned long long* d_keys_s = cv.take<unsigned long long>(N);
  int* d_idx = cv.take<int>(N + 1);
  int* d_idx_s = cv.take<int>(N + 1);
  int* d_flags = cv.take<int>(N + 1);
  int* d_pos = cv.take<int>(N + 1);
  int* d_starts = cv.take<int>(N + 1);
  int* d_keep = cv.take<int>(N + 1);
  void* h_mf = nullptr;
  GB_CHECK(gb_ctx_pinned(ctx, sizeof(MergeFrame) * (size_t)K, &h_mf));
  memcpy(h_mf, mf.data(), sizeof(MergeFrame) * (size_t)K);
  GB_CUDA(cudaMemcpyAsync(d_mf, h_mf, sizeof(MergeFrame) * (size_t)K, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemsetAsync(d_cnt, 0, 256, st));
  const int tb = 256, gb = (n + tb - 1) / tb;
  k_merge_transform<<<gb, tb, 0, st>>>(K, d_mf, n, d_pts, d_cov);
  k_grid_keys<<<gb, tb, 0, st>>>(n, d_pts, 1.0 / resolution, d_keys, d_idx);
  size_t tmp = cub_b;
  GB_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, tmp, d_keys, d_keys_s, d_idx, d_idx_s, n, 0, 64, st));
  k_grid_flags<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags);
  tmp = cub_b;
  GB_CUDA(cub::DeviceScan::InclusiveSum(d_cub, tmp, d_flags, d_pos, n, st));
  k_copy_last_pos<<<1, 1, 0, st>>>(n, d_pos, d_cnt);  // V
  k_grid_starts<<<gb, tb, 0, st>>>(n, d_keys_s, d_flags, d_pos, d_starts);
  k_merge_means<<<(n + 127) / 128, 128, 0, st>>>(d_cnt, d_starts, d_idx_s, d_pts, d_cov, d_vpts, d_vcov);
  // thinning to target_num_points
  k_merge_hash_keys<<<gb, tb, 0, st>>>(n, d_cnt, seed, d_keys);
  tmp = cub_b;
  GB_CUDA(cub::DeviceRadixSort::SortKeys(d_cub, tmp, d_keys, d_keys_s, n, 0, 64, st));
  k_merge_keep<<<gb, tb, 0, st>>>(n, d_cnt, target, d_keys_s, seed, d_keep);
  tmp = cub_b;
  GB_CUDA(cub::DeviceScan::InclusiveSum(d_cub, tmp, d_keep, d_pos, n, st));
  int M = 0;
  GB_CUDA(cudaMemcpyAsync(&M, d_pos + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  ctx->launches += 12;
  *num_out = (size_t)M;
  if (M == 0) return GB_OK;
  const size_t c0 = align_up(16 * (size_t)M, 256), c2 = align_up(4 * (size_t)M, 256);
  float4* s0 = (float4*)staged;
  float4* s1 = (float4*)(staged + c0);
  float* s2 = (float*)(staged + 2 * c0);
  k_merge_emit<<<gb, tb, 0, st>>>(n, d_keep, d_pos, d_vpts, d_vcov, d_pts /* reused: emitted points */, d_ocov, s0, s1, s2);
  GB_CUDA(cudaGetLastError());
  ctx->launches++;
  if (cloud_out) {
    const size_t ctotal = 2 * c0 + c2;
    const size_t bperm = align_up(sizeof(int) * (size_t)M, 256);
    cloud_out->n = (size_t)M;
    GB_CUDA(gb_dev_malloc(ctx->device, ctotal + 2 * bperm, &cloud_out->base));
    cloud_out->bytes = ctotal + 2 * bperm;
    char* d = (char*)cloud_out->base;
    cloud_out->p0 = (float4*)d; cloud_out->p1 = (float4*)(d + c0); cloud_out->p2 = (float*)(d + 2 * c0); cloud_out->normals = nullptr;
    cloud_out->perm = (int*)(d + ctotal); cloud_out->inv_perm = (int*)(d + ctotal + bperm);
    GB_CHECK(gb_cloud_reorder_impl(ctx, cloud_out, staged, c0, c0, c2, 0));
  }
  if (out_xyzw) GB_CUDA(cudaMemcpyAsync(out_xyzw, d_pts, sizeof(double4) * (size_t)M, cudaMemcpyDeviceToHost, st));
  if (out_cov4x4) GB_CUDA(cudaMemcpyAsync(out_cov4x4, d_ocov, sizeof(double) * 16 * (size_t)M, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return GB_OK;
}

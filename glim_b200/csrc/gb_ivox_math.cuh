// gb_ivox_math.cuh -- the correspondence search of the GICP sweep (k_gicp_sweep, gb_kernels_vgicp.cu) on a device iVox, kept
// free of anything that only exists on the device so that the SAME TEXT also compiles for the host:
// tests/cpp/ivox_search_host.cpp builds it with g++ and tests/test_ivox_host.py checks it against the numpy restatement of the
// rule (tests/ivox_oracle.py) on the CPU-only box.  The rule is written once, in include/glim_b200.h (gb_gicp_factor_create).
#pragma once
#include "gb_vgicp_math.cuh"  // GB_HD, gb_coord, gb_hash, PoseF, transform

#ifndef __CUDACC__
struct int2 { int x, y; };
// the host build compiles with -ffp-contract=off: plain operations are the round-to-nearest intrinsics
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
#endif

namespace {

// The k-th voxel offset of the search ([EXT]: gtsam_points' neighbour tables are not vendored).  neighbor_voxel_mode m searches
// k = 0 .. m - 1:
//   0       the centre;
//   1 - 6   the faces -x +x -y +y -z +z;
//   7 - 18  the edges: the zero axis x, then y, then z; the two other axes' signs (--, -+, +-, ++) in axis order;
//   19 - 26 the corners: (dx, dy, dz) in {-1, +1}^3, lexicographic.
GB_HD void ivox_offset(int k, int& dx, int& dy, int& dz) {
  dx = 0; dy = 0; dz = 0;
  if (k == 0) return;
  if (k < 7) {
    const int f = k - 1, s = (f & 1) ? 1 : -1;
    if (f < 2) dx = s; else if (f < 4) dy = s; else dz = s;
    return;
  }
  if (k < 19) {
    const int e = k - 7, zero = e / 4;
    const int s1 = (e & 2) ? 1 : -1, s2 = (e & 1) ? 1 : -1;
    if (zero == 0) { dy = s1; dz = s2; } else if (zero == 1) { dx = s1; dz = s2; } else { dx = s1; dy = s2; }
    return;
  }
  const int c = k - 19;
  dx = (c & 4) ? 1 : -1; dy = (c & 2) ? 1 : -1; dz = (c & 1) ? 1 : -1;
}

// linear-probing lookup of voxel (cx, cy, cz) in the iVox's table: its index, -1 if absent
GB_HD int ivox_find(const int4* __restrict__ buckets, uint32_t mask, int max_scan, int cx, int cy, int cz) {
  const uint32_t h = gb_hash(cx, cy, cz);
  for (int i = 0; i < max_scan; i++) {
    const int4 b = buckets[(h + (uint32_t)i) & mask];
    if (b.w < 0) return -1;
    if (b.x == cx && b.y == cy && b.z == cz) return b.w;
  }
  return -1;
}

// The correspondence of a transformed source point q: the stored point nearest to q among the points of the searched voxels,
// if its squared distance is below max_d2; -1 otherwise.  Distances are fp32 in one fixed order,
// d2 = (dx * dx + dy * dy) + dz * dz with d = p - q, never contracted; a tie keeps the earlier offset, then the earlier slot.
// A NaN q keys to voxel (0, 0, 0) and its distances are NaN: it never matches.
GB_HD int ivox_nearest(const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells, const float4* __restrict__ points,
                       int num_offsets, float inv_res, float max_d2, float qx, float qy, float qz) {
  const int cx = gb_coord(qx, inv_res), cy = gb_coord(qy, inv_res), cz = gb_coord(qz, inv_res);
  int best = -1;
  float best_d2 = max_d2;
  for (int k = 0; k < num_offsets; k++) {
    int dx, dy, dz;
    ivox_offset(k, dx, dy, dz);
    // wrapping sums: a saturated coordinate (a point far outside the key range) finds nothing
    const int v = ivox_find(buckets, mask, max_scan, (int)((uint32_t)cx + (uint32_t)dx), (int)((uint32_t)cy + (uint32_t)dy), (int)((uint32_t)cz + (uint32_t)dz));
    if (v < 0) continue;
    const int2 c = cells[v];
    for (int s = 0; s < c.y; s++) {
      const float4 p = points[3 * (size_t)(c.x + s)];
      const float ex = __fsub_rn(p.x, qx), ey = __fsub_rn(p.y, qy), ez = __fsub_rn(p.z, qz);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
      if (d2 < best_d2) { best_d2 = d2; best = c.x + s; }
    }
  }
  return best;
}

}  // namespace

// gb_grid_math.cuh -- the correspondence search of the GICP and ICP sweeps on a device point grid (k_gicp_grid_sweep,
// k_icp_grid_sweep, gb_kernels_gicp.cu),
// kept free of anything that only exists on the device so that the SAME TEXT also compiles for the host:
// tests/cpp/grid_search_host.cpp builds it with g++ and tests/test_grid_host.py checks it against the numpy restatement of the
// rule (tests/grid_oracle.py) on the CPU-only box.  The rule is written once, in include/glim_b200.h (gb_point_grid_build,
// gb_gicp_grid_factor_create).
#pragma once
#include "gb_ivox_math.cuh"  // GB_HD, gb_coord, gb_lookup, point_d2, the host shims of the fp32 intrinsics

#ifndef __CUDACC__
#include <string.h>
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, sizeof(i)); return i; }
#endif

namespace {

// The largest search half-width gb_gicp_grid_factor_create accepts: (2 * 8 + 1)^3 = 4913 cells per query.
constexpr int kGridMaxHalfWidth = 8;

// The search half-width m: the smallest integer for which every stored point p with fp32 d2(p, q) < max_d2 lies in a cell
// c(q) + o, o in [-m, m]^3.  inv = (float)(1 / cell_size); key_extent K >= max(|k|, |k + 1|) over every axis k of every cell.
//
// Proof, per axis, with u = 2^-24 (fp32 round to nearest) and exact real arithmetic on the fp32 values:
//   1. d2 = ((ex*ex + ey*ey) + ez*ez) rounded at each step, with ex = fl(p.x - q.x).  Every term is >= 0 and rounding is
//      monotone, so d2 >= fl(ex*ex); max_d2 is a float, so fl(ex*ex) < max_d2 implies ex*ex < max_d2.  Hence
//      |ex| < sqrt(max_d2), and since a subtraction errs by at most u of its result, |p.x - q.x| < D = sqrt(max_d2) / (1 - u).
//      (A NaN or infinite d2 fails d2 < max_d2: such a pair never matches.)
//   2. The cell of p is floor(fl(p.x * inv)) with fl(p.x * inv) in [k, k + 1), so |fl(p.x * inv)| <= K and
//      |p.x * inv| <= A_p = K / (1 - u).  Then |q.x * inv| <= A_q = A_p + D * inv.
//   3. A product errs by at most u of its exact value (plus 2^-149 below the normal range), so
//      |fl(p.x * inv) - fl(q.x * inv)| <= D * inv + u * (A_p + A_q) + 2^-148 = W.
//   4. |floor(a) - floor(b)| < |a - b| + 1 <= W + 1, so the cells differ by at most ceil(W) (an integer below W + 1).
// W is evaluated in fp64, whose own rounding (a few 1e-16 relative) is covered by the factor 1 + 2^-40.  The rounding of
// 1 / cell_size needs no term: every key, of stored and query points alike, is formed with the same fp32 inv.
// Returns ceil(W), or kGridMaxHalfWidth + 1 when W exceeds kGridMaxHalfWidth (or is not finite).  Host code: the factor's
// creation computes it once.
inline int grid_half_width(float inv, float max_d2, int key_extent) {
  const double u = 1.0 / 16777216.0;
  const double D = sqrt((double)max_d2) / (1.0 - u);
  const double Ap = (double)key_extent / (1.0 - u);
  const double Aq = Ap + D * (double)inv;
  const double W = (D * (double)inv + u * (Ap + Aq) + 0x1p-148) * (1.0 + 0x1p-40);
  if (!(W <= (double)kGridMaxHalfWidth)) return kGridMaxHalfWidth + 1;
  return (int)ceil(W);
}

// The original index of a grid record (slot 2.z holds its bits).
GB_HD int grid_record_index(const float4* __restrict__ points, int r) { return __float_as_int(points[3 * (size_t)r + 2].z); }

// The correspondence of a transformed source point q: the stored point with the smallest fp32 d2 = point_d2(p, q) among the
// cells c(q) + o, o in [-m, m]^3, if d2 < max_d2; ties go to the smaller original index.  With m from grid_half_width this is
// the brute-force argmin over every stored point, whatever the visiting order.  Returns the record, -1 for none.  A NaN q keys
// to cell (0, 0, 0) and its distances are NaN: it never matches; a saturated coordinate wraps out of the key range and finds
// nothing.
GB_HD int grid_nearest(const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells, const float4* __restrict__ points,
                       int m, float inv, float max_d2, float qx, float qy, float qz) {
  const int cx = gb_coord(qx, inv), cy = gb_coord(qy, inv), cz = gb_coord(qz, inv);
  int best = -1;
  float best_d2 = max_d2;
  for (int ox = -m; ox <= m; ox++) {
    for (int oy = -m; oy <= m; oy++) {
      for (int oz = -m; oz <= m; oz++) {
        const int v = gb_lookup(buckets, mask, max_scan, (int)((uint32_t)cx + (uint32_t)ox), (int)((uint32_t)cy + (uint32_t)oy), (int)((uint32_t)cz + (uint32_t)oz));
        if (v < 0) continue;
        const int2 c = cells[v];
        for (int s = 0; s < c.y; s++) {
          const int r = c.x + s;
          const float d2 = point_d2(points[3 * (size_t)r], qx, qy, qz);
          if (d2 < best_d2) {
            best_d2 = d2;
            best = r;
          } else if (d2 == best_d2 && best >= 0 && grid_record_index(points, r) < grid_record_index(points, best)) {
            best = r;
          }
        }
      }
    }
  }
  return best;
}

// Every stored point p with fp32 point_d2(p, q) < max_d2: visit(record) for each, cells in offset order and
// the points of a cell in ascending original index.  With m from grid_half_width this is exactly the brute-force set (the proof
// above bounds every such point, not only the nearest).  The FPFH neighbourhood of gb_cloud_estimate_fpfh.
template <typename Visit>
GB_HD void grid_within(const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells, const float4* __restrict__ points,
                       int m, float inv, float max_d2, float qx, float qy, float qz, Visit&& visit) {
  const int cx = gb_coord(qx, inv), cy = gb_coord(qy, inv), cz = gb_coord(qz, inv);
  for (int ox = -m; ox <= m; ox++) {
    for (int oy = -m; oy <= m; oy++) {
      for (int oz = -m; oz <= m; oz++) {
        const int v = gb_lookup(buckets, mask, max_scan, (int)((uint32_t)cx + (uint32_t)ox), (int)((uint32_t)cy + (uint32_t)oy), (int)((uint32_t)cz + (uint32_t)oz));
        if (v < 0) continue;
        const int2 c = cells[v];
        for (int s = 0; s < c.y; s++) {
          const int r = c.x + s;
          const float d2 = point_d2(points[3 * (size_t)r], qx, qy, qz);
          if (d2 < max_d2) visit(r);
        }
      }
    }
  }
}

}  // namespace

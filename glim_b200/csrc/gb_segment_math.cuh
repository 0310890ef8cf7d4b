// gb_segment_math.cuh -- the per-point and per-pair arithmetic of the map segmentation (gb_concat_frames, gb_region_growing,
// gb_kernels_segment.cu), and the posed frame list that gb_concat_frames shares with gb_merge_frames, the map insert and the
// plane selection (gb_frame, gb_frame_of), kept free of anything that only exists on the device so that the SAME TEXT also
// compiles for the host: tests/cpp/segment_math_host.cpp builds it with g++ -ffp-contract=off and tests/test_segment_host.py
// checks it against the numpy restatement of the rules (tests/segment_oracle.py).  The rules are written once, in
// include/glim_b200.h.
#pragma once
#include "gb_grid_math.cuh"  // GB_HD, gb_coord, point_d2, grid_within, the fp32 intrinsics' host shims
#include "gb_cov_math.cuh"   // the fp64 intrinsics' host shims

// The descriptor of frame k of a posed frame list (gb_frame_table): the cloud's stored planes, normals and storage order, its
// point count, its first point in the concatenation of the list, the caller's index of the frame, and the rows of its 3x4 pose.
struct gb_frame {
  const float4* p0;
  const float4* p1;
  const float* p2;
  const float4* normals;
  const int* inv_perm;
  int n, offset, index;
  double T[12];
};

namespace {

// The frame of K (K >= 1) that holds point g of the concatenation: the last whose first point is at or before g.  A frame
// with no points shares its offset with the next one, so it never holds g.
GB_HD int gb_frame_of(const gb_frame* frames, int K, int g) {
  int a = 0, b = K - 1;
  while (a < b) {
    const int mid = (a + b + 1) / 2;
    if (frames[mid].offset <= g) a = mid; else b = mid - 1;
  }
  return a;
}

// The 21-bit key range of every grid: a point takes part in a search of a grid of fp32 cell inverse inv iff it is finite and
// each gb_coord(x, inv) lies in [-2^20, 2^20) (the points without a key are in no cell of the grid).
GB_HD bool seg_keyed(float x, float y, float z, float inv) {
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
  const int k[3] = {gb_coord(x, inv), gb_coord(y, inv), gb_coord(z, inv)};
  for (int a = 0; a < 3; a++)
    if (k[a] < -(1 << 20) || k[a] >= (1 << 20)) return false;
  return true;
}

// The normal test of an edge: (nx_i nx_j + ny_i ny_j) + nz_i nz_j in fp64 from the fp32 normals, each operation rounded, at
// least cos_t (signed; a NaN dot never joins).
GB_HD bool seg_normals_join(float ax, float ay, float az, float bx, float by, float bz, double cos_t) {
  const double d = __dadd_rn(__dadd_rn(__dmul_rn((double)ax, (double)bx), __dmul_rn((double)ay, (double)by)), __dmul_rn((double)az, (double)bz));
  return d >= cos_t;
}

// The seed order: (fp32 point_d2 of p to q, original index i) packed so that the smaller key is the nearer point, ties to the
// smaller index; ~0 for a point that is not finite.  d2 >= 0 (or +inf), so its bits order as unsigned integers.
GB_HD unsigned long long seg_seed_key(float4 p, float qx, float qy, float qz, int i) {
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return ~0ull;
  return ((unsigned long long)(uint32_t)__float_as_int(point_d2(p, qx, qy, qz)) << 32) | (uint32_t)i;
}

// A point's normal rotated into the world frame: n' = R n, row r as (R_r0 nx + R_r1 ny) + R_r2 nz in un-contracted fp64 (T:
// the rows of the 3x4 pose [R | t], gb_frame::T), stored fp32, not renormalised.
GB_HD void seg_rotate_normal(const double* T, float nx, float ny, float nz, float* out) {
  for (int r = 0; r < 3; r++)
    out[r] = (float)__dadd_rn(__dadd_rn(__dmul_rn(T[4 * r], (double)nx), __dmul_rn(T[4 * r + 1], (double)ny)), __dmul_rn(T[4 * r + 2], (double)nz));
}

// The window test of gb_concat_frames: floor(q * (1.0 / cell_size)) in fp64 within [lo, hi] on every axis; never for a
// non-finite q.
GB_HD bool seg_in_window(const double* q, double inv, const int* lo, const int* hi) {
  for (int a = 0; a < 3; a++) {
    if (!isfinite(q[a])) return false;
    const double k = floor(__dmul_rn(q[a], inv));
    if (k < (double)lo[a] || k > (double)hi[a]) return false;
  }
  return true;
}

// Union-find over original indices with parent[x] <= x for every x (a root is its own parent).  Roots only ever gain a
// smaller parent, so the root of a component is its minimum index whatever the order of the hooks (ECL-CC).  On the device
// many threads hook at once: a link is a compare-and-swap of a root's own entry, and a reader may see any ancestor, which is
// always a valid shortcut.
GB_HD int seg_cas(int* a, int expected, int desired) {
#ifdef __CUDACC__
  return atomicCAS(a, expected, desired);
#else
  const int old = *a;
  if (old == expected) *a = desired;
  return old;
#endif
}

GB_HD int seg_find(const int* parent, int x) {
  const volatile int* p = parent;
  int y = p[x];
  while (y != x) {
    x = y;
    y = p[x];
  }
  return x;
}

// joins the components of a and b: the larger root goes under the smaller
GB_HD void seg_hook(int* parent, int a, int b) {
  int ra = seg_find(parent, a), rb = seg_find(parent, b);
  while (ra != rb) {
    if (ra > rb) { const int t = ra; ra = rb; rb = t; }
    const int old = seg_cas(&parent[rb], rb, ra);
    if (old == rb) return;
    rb = seg_find(parent, old);  // rb gained a parent meanwhile: retry from its new root
    ra = seg_find(parent, ra);
  }
}

// True iff some stored point of an R record (flag[original index]) lies within max_d2 of q: grid_within's search with an
// early exit.  Only its existence matters, so the visiting order does not.
GB_HD bool seg_grid_any(const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells, const float4* __restrict__ points,
                        int m, float inv, float max_d2, float qx, float qy, float qz, const int* __restrict__ flag) {
  const int cx = gb_coord(qx, inv), cy = gb_coord(qy, inv), cz = gb_coord(qz, inv);
  for (int ox = -m; ox <= m; ox++) {
    for (int oy = -m; oy <= m; oy++) {
      for (int oz = -m; oz <= m; oz++) {
        const int v = gb_lookup(buckets, mask, max_scan, (int)((uint32_t)cx + (uint32_t)ox), (int)((uint32_t)cy + (uint32_t)oy), (int)((uint32_t)cz + (uint32_t)oz));
        if (v < 0) continue;
        const int2 c = cells[v];
        for (int s = 0; s < c.y; s++) {
          const int r = c.x + s;
          if (flag[grid_record_index(points, r)] && point_d2(points[3 * (size_t)r], qx, qy, qz) < max_d2) return true;
        }
      }
    }
  }
  return false;
}

}  // namespace

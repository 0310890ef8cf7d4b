// Host build of the sweep kernels' per-point arithmetic (glim_b200/csrc/gb_vgicp_math.cuh -- the SAME text the kernels compile)
// driven by a scalar emulation of k_vgicp_sweep3's item structure: rounds of 512 points, lookup -> compaction in point order ->
// lane k % 32 takes hit k -> transposing warp reduce-scatter in fp32 -> fp64 accumulation per item.  TEST INFRASTRUCTURE: built
// by tests/test_kernel_math_host.py with g++ and compared with the CPU oracle on the CPU-only box; nothing in the product links it.
#include <stdlib.h>
#include <string.h>

#include "../../glim_b200/csrc/gb_vgicp_math.cuh"

namespace {

// warp_reduce_scatter32 of the kernel, lanes as an array index: on return v[l][0] = sum over lanes of v[.][l]
void reduce_scatter32(float (*v)[32]) {
  for (int step = 16; step >= 1; step >>= 1) {
    float nv[32][32];
    for (int lane = 0; lane < 32; lane++) {
      const bool upper = (lane & step) != 0;
      const int other = lane ^ step;
      const bool oupper = (other & step) != 0;
      for (int j = 0; j < step; j++) {
        const float keep = upper ? v[lane][j + step] : v[lane][j];
        const float recv = oupper ? v[other][j] : v[other][j + step];  // what the partner sends
        nv[lane][j] = keep + recv;
      }
    }
    for (int lane = 0; lane < 32; lane++)
      for (int j = 0; j < step; j++) v[lane][j] = nv[lane][j];
  }
}

}  // namespace

// planes as in gb_cloud: p0 = {x y z c00}, p1 = {c01 c02 c11 c12}, p2 = c22, normals4 = {nx ny nz 0} or NULL;
// voxels: 3 float4 per voxel.  T_eval == NULL: linearize at T_lin; else error mode (inliers at T_lin, residuals at T_eval).
// acc29: upper triangle of H_tt (21, row-major) | b_t (6) | error | inlier count.  corr[i] = voxel index, -1 miss, -2 gate.
extern "C" int km_sweep(int n, const float* p0, const float* p1, const float* p2, const float* normals4, const int* buckets, unsigned mask, int max_scan,
                        const float* voxels, float inv_res, const double* T_lin, const double* T_eval, int chunk, double* acc29, int* corr) {
  const float4* P0 = reinterpret_cast<const float4*>(p0);
  const float4* P1 = reinterpret_cast<const float4*>(p1);
  const float4* NR = reinterpret_cast<const float4*>(normals4);
  const int4* B = reinterpret_cast<const int4*>(buckets);
  const float4* V = reinterpret_cast<const float4*>(voxels);
  const PoseF P = pose_from_colmajor(T_lin);
  const PoseF Pe = T_eval ? pose_from_colmajor(T_eval) : P;
  for (int k = 0; k < 29; k++) acc29[k] = 0.0;
  if (chunk <= 0) chunk = 2048;
  static float acc[32][32];
  int* qi = (int*)malloc(sizeof(int) * 512);
  int* qv = (int*)malloc(sizeof(int) * 512);
  for (int first = 0; first < n; first += chunk) {
    const int item_end = first + chunk < n ? first + chunk : n;
    memset(acc, 0, sizeof(acc));
    for (int wb = first; wb < item_end; wb += 512) {
      const int we = wb + 512 < item_end ? wb + 512 : item_end;
      int nq = 0;
      for (int i = wb; i < we; i++) {  // phase A
        float qx, qy, qz;
        transform(P, P0[i].x, P0[i].y, P0[i].z, qx, qy, qz);
        const int v = gb_lookup(B, mask, max_scan, gb_coord(qx, inv_res), gb_coord(qy, inv_res), gb_coord(qz, inv_res));
        if (corr) corr[i] = v;
        if (v >= 0) { qi[nq] = i; qv[nq] = v; nq++; }
      }
      for (int k = 0; k < nq; k++) {  // phase B: lane k % 32 takes hit k
        const int i = qi[k];
        const float4 v0 = V[3 * (size_t)qv[k] + 0], v1 = V[3 * (size_t)qv[k] + 1], v2 = V[3 * (size_t)qv[k] + 2];
        if (NR && !surface_ok(P, NR[i], v0.w, v1.x, v1.y, v1.z, v1.w, v2.x)) {
          if (corr) corr[i] = -2;
          continue;
        }
        if (T_eval) accumulate_hit<1>(acc[k & 31], Pe, P0[i], P1[i], p2[i], v0, v1, v2);
        else accumulate_hit<0>(acc[k & 31], Pe, P0[i], P1[i], p2[i], v0, v1, v2);
      }
    }
    reduce_scatter32(acc);
    for (int l = 0; l < 29; l++) acc29[l] += (double)acc[l][0];
  }
  free(qi);
  free(qv);
  return 0;
}

// slab row element -> index in the 122-double record (the mapping pair_push uses)
extern "C" int km_slab_to_record(int e) { return slab_to_record(e); }
extern "C" int km_coord(float p, float inv_res) { return gb_coord(p, inv_res); }
extern "C" unsigned km_hash(int x, int y, int z) { return gb_hash(x, y, z); }

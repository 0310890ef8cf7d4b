// Host build of the grid GICP sweep's correspondence search (glim_b200/csrc/gb_grid_math.cuh, the text k_gicp_grid_sweep
// compiles): tests/test_grid_host.py compiles this with g++ -ffp-contract=off and compares it with the numpy restatement of the
// rule (tests/grid_oracle.py).
#include "../../glim_b200/csrc/gb_grid_math.cuh"

extern "C" {

// corr[i] = record of source point i's correspondence at T (16 doubles, column-major), -1 for none
void gs_search(int n, const float* xyz /* n x 3 */, const double* T, const int4* buckets, unsigned mask, int max_scan, const int2* cells,
               const float4* points, int m, float inv, float max_d2, int* corr) {
  const PoseF P = pose_from_colmajor(T);
  for (int i = 0; i < n; i++) {
    float qx, qy, qz;
    transform(P, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], qx, qy, qz);
    corr[i] = grid_nearest(buckets, mask, max_scan, cells, points, m, inv, max_d2, qx, qy, qz);
  }
}

// the same search for queries given in the target frame (no transform): adversarial q placed bit by bit
void gs_search_q(int n, const float* q /* n x 3 */, const int4* buckets, unsigned mask, int max_scan, const int2* cells, const float4* points, int m,
                 float inv, float max_d2, int* corr) {
  for (int i = 0; i < n; i++) corr[i] = grid_nearest(buckets, mask, max_scan, cells, points, m, inv, max_d2, q[3 * i], q[3 * i + 1], q[3 * i + 2]);
}

int gs_half_width(float inv, float max_d2, int key_extent) { return grid_half_width(inv, max_d2, key_extent); }

}  // extern "C"

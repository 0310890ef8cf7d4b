// Host build of the GICP sweep's correspondence search (glim_b200/csrc/gb_ivox_math.cuh, the text k_gicp_sweep compiles):
// tests/test_ivox_host.py compiles this with g++ -ffp-contract=off and compares it with the numpy restatement of the rule.
#include "../../glim_b200/csrc/gb_ivox_math.cuh"

extern "C" {

// corr[i] = record of source point i's correspondence at T (16 doubles, column-major), -1 for none
void ivs_search(int n, const float* xyz /* n x 3 */, const double* T, const int4* buckets, unsigned mask, int max_scan, const int2* cells,
                const float4* points, int num_offsets, float inv_res, float max_d2, int* corr) {
  const PoseF P = pose_from_colmajor(T);
  for (int i = 0; i < n; i++) {
    float qx, qy, qz;
    transform(P, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], qx, qy, qz);
    corr[i] = ivox_nearest(buckets, mask, max_scan, cells, points, num_offsets, inv_res, max_d2, qx, qy, qz);
  }
}

void ivs_offset(int k, int* d) { ivox_offset(k, d[0], d[1], d[2]); }

}  // extern "C"

// Host build of the global-registration arithmetic (glim_b200/csrc/gb_global_math.cuh, the text the kernels of
// gb_kernels_global.cu compile): tests/test_global_host.py compiles this with g++ -ffp-contract=off and compares it with the numpy
// restatement (tests/global_oracle.py).
#include "../../glim_b200/csrc/gb_global_math.cuh"

extern "C" {

// pair features f (n x 3) and bins (n x 3) of n pairs (positions and normals n x 3 each)
void gm_pairs(int n, const double* ps, const double* ns, const double* pt, const double* nt, double* f, int* b) {
  for (int i = 0; i < n; i++) {
    fpfh_pair(ps + 3 * i, ns + 3 * i, pt + 3 * i, nt + 3 * i, f + 3 * i);
    fpfh_bins(f + 3 * i, b + 3 * i);
  }
}

// the samples of hypotheses h0 .. h0 + count - 1 (count x 3)
void gm_samples(unsigned long long seed, int h0, int count, int ns, int* s) {
  for (int k = 0; k < count; k++) ransac_sample(seed, h0 + k, ns, s + 3 * k);
}

// T (16, column-major) from source a and target b (3 x 3 each); returns 0 for an invalid sample
int gm_pose(const double* a, const double* b, int dof, double* T) { return ransac_pose(a, b, dof, T) ? 1 : 0; }

// the radius neighbours of query i over a point grid, as k_fpfh_spfh visits them (records), up to cap; returns their number
int gm_within(const int4* buckets, unsigned mask, int max_scan, const int2* cells, const float4* points, int m, float inv, float max_d2, float qx, float qy,
              float qz, int cap, int* out) {
  int k = 0;
  grid_within(buckets, mask, max_scan, cells, points, m, inv, max_d2, qx, qy, qz, [&](int r) {
    if (k < cap) out[k] = r;
    k++;
  });
  return k;
}

// inlier count of a pose (16 doubles, column-major) over n source points against a grid's table
int gm_inliers(const double* T, int n, const float* xyz, const int4* buckets, unsigned mask, int max_scan, float inv) {
  const PoseF P = pose_from_colmajor(T);
  int c = 0;
  for (int i = 0; i < n; i++) c += ransac_inlier(P, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], buckets, mask, max_scan, inv) ? 1 : 0;
  return c;
}

}  // extern "C"
